// Row-wise / memory-bound kernels of the phenaki hot path (sm_90a).
// Every kernel cites the reference code it replaces (paths relative to
// /root/reference/phenaki_pytorch/).  All are HBM/L2-bound: coalesced 16-byte accesses,
// no tensor cores on purpose.
#include "phk_common.cuh"

namespace phk {

// ------------------------------------------------------------------------------------------
// LayerNorm (attention.py:29-36, :48, :308): two-pass mean / variance, eps 1e-5, fp32.
// Warp-per-row fast path for dim % 128 == 0 && dim <= 1024; block-per-row otherwise.
// ------------------------------------------------------------------------------------------
template <int VEC /* float4 per lane */>
__global__ void __launch_bounds__(256) ln_warp_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                      const float* __restrict__ b, void* __restrict__ out,
                                                      __nv_bfloat16* __restrict__ raw, int64_t rows, int dim,
                                                      int out_bf16, int64_t seg_len, int64_t seg_stride,
                                                      int64_t seg_off) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  // seg_len > 0: scatter (the map places the OUTPUT row); seg_len < 0: gather (the map picks the INPUT row)
  const int64_t sl = seg_len < 0 ? -seg_len : seg_len;
  const int64_t mrow = sl > 0 ? (row / sl) * seg_stride + seg_off + row % sl : row;
  const int64_t orow = seg_len < 0 ? row : mrow;
  const float4* xr = reinterpret_cast<const float4*>(x + (seg_len < 0 ? mrow : row) * dim);
  float4 v[VEC];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    v[j] = xr[lane + 32 * j];
    s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
  }
  const float mean = warp_sum(s) / (float)dim;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    float a = v[j].x - mean, bb = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
    q += (a * a + bb * bb) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)dim + 1e-5f);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const float4* b4 = reinterpret_cast<const float4*>(b);
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const int c4 = lane + 32 * j;
    const float4 gg = g4[c4], bb = b4[c4];
    float4 o;
    o.x = (v[j].x - mean) * rstd * gg.x + bb.x;
    o.y = (v[j].y - mean) * rstd * gg.y + bb.y;
    o.z = (v[j].z - mean) * rstd * gg.z + bb.z;
    o.w = (v[j].w - mean) * rstd * gg.w + bb.w;
    if (out_bf16) {
      uint2 p = make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
      reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + orow * dim)[c4] = p;
    } else {
      reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + orow * dim)[c4] = o;
    }
    if (raw) {
      uint2 p = make_uint2(pack_bf16x2(v[j].x, v[j].y), pack_bf16x2(v[j].z, v[j].w));
      reinterpret_cast<uint2*>(raw + orow * dim)[c4] = p;
    }
  }
}

__global__ void __launch_bounds__(256) ln_block_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                       const float* __restrict__ b, void* __restrict__ out,
                                                       __nv_bfloat16* __restrict__ raw, int dim, int out_bf16,
                                                       int64_t seg_len, int64_t seg_stride, int64_t seg_off) {
  pdl_prologue();
  extern __shared__ float srow[];
  __shared__ float red[32];
  const int64_t row = blockIdx.x;
  const int64_t sl = seg_len < 0 ? -seg_len : seg_len;
  const int64_t mrow = sl > 0 ? (row / sl) * seg_stride + seg_off + row % sl : row;
  const int64_t orow = seg_len < 0 ? row : mrow;
  const float* xr = x + (seg_len < 0 ? mrow : row) * dim;
  float s = 0.f;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) { float t = xr[i]; srow[i] = t; s += t; }
  const float mean = block_sum(s, red) / (float)dim;
  float q = 0.f;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) { float d = srow[i] - mean; q += d * d; }
  const float rstd = rsqrtf(block_sum(q, red) / (float)dim + 1e-5f);
  for (int i = threadIdx.x; i < dim; i += blockDim.x) {
    const float o = (srow[i] - mean) * rstd * g[i] + b[i];
    if (out_bf16) reinterpret_cast<__nv_bfloat16*>(out)[orow * dim + i] = __float2bfloat16_rn(o);
    else reinterpret_cast<float*>(out)[orow * dim + i] = o;
    if (raw) raw[orow * dim + i] = __float2bfloat16_rn(srow[i]);
  }
}

// ------------------------------------------------------------------------------------------
// Patchify + LayerNorm(K) (cvivit.py:273-275 / 280-282).  One CTA per token; the token's K
// pixels are gathered as p2-float contiguous runs (128 B for p2=32) straight from the
// (B,C,F,H,W) video -- the single HBM-visible read of the encoder -- into shared memory,
// normalised in place and written as one dense row of the GEMM A operand.
// ------------------------------------------------------------------------------------------
template <bool VEC4>
__global__ void __launch_bounds__(256) patchify_ln_kernel(const float* __restrict__ video, int C, int F, int H,
                                                          int W, int f0, int nt, int pt, int p1, int p2,
                                                          const float* __restrict__ g, const float* __restrict__ b,
                                                          void* __restrict__ out, int out_bf16) {
  pdl_prologue();
  extern __shared__ float srow[];
  __shared__ float red[32];
  const int hh = H / p1, ww = W / p2;
  int tok = blockIdx.x;
  const int wi = tok % ww; tok /= ww;
  const int hi = tok % hh; tok /= hh;
  const int ti = tok % nt;
  const int bi = tok / nt;
  const int K = C * pt * p1 * p2;
  const int64_t plane = (int64_t)H * W;
  const float* base = video + ((int64_t)bi * C * F + f0 + (int64_t)ti * pt) * plane + (int64_t)hi * p1 * W + wi * p2;
  float s = 0.f;
  if (VEC4) {
    const int runs = p2 >> 2;  // float4 per patch row
    for (int i = threadIdx.x; i < (K >> 2); i += blockDim.x) {
      const int dx4 = i % runs;
      int r = i / runs;  // (c, dt, dy)
      const int dy = r % p1; r /= p1;
      const int dt = r % pt;
      const int c = r / pt;
      const float4 v = __ldg(reinterpret_cast<const float4*>(base + ((int64_t)c * F + dt) * plane + (int64_t)dy * W) + dx4);
      reinterpret_cast<float4*>(srow)[i] = v;
      s += (v.x + v.y) + (v.z + v.w);
    }
  } else {
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
      const int dx = i % p2;
      int r = i / p2;
      const int dy = r % p1; r /= p1;
      const int dt = r % pt;
      const int c = r / pt;
      const float v = __ldg(base + ((int64_t)c * F + dt) * plane + (int64_t)dy * W + dx);
      srow[i] = v;
      s += v;
    }
  }
  const float mean = block_sum(s, red) / (float)K;
  float q = 0.f;
  for (int i = threadIdx.x; i < K; i += blockDim.x) { const float d = srow[i] - mean; q += d * d; }
  const float rstd = rsqrtf(block_sum(q, red) / (float)K + 1e-5f);
  const int64_t orow = (int64_t)blockIdx.x * K;
  if (VEC4) {
    for (int i = threadIdx.x; i < (K >> 2); i += blockDim.x) {
      const float4 v = reinterpret_cast<float4*>(srow)[i];
      const float4 gg = __ldg(reinterpret_cast<const float4*>(g) + i);
      const float4 bb = __ldg(reinterpret_cast<const float4*>(b) + i);
      float4 o;
      o.x = (v.x - mean) * rstd * gg.x + bb.x;
      o.y = (v.y - mean) * rstd * gg.y + bb.y;
      o.z = (v.z - mean) * rstd * gg.z + bb.z;
      o.w = (v.w - mean) * rstd * gg.w + bb.w;
      if (out_bf16)
        reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + orow)[i] =
            make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
      else
        reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + orow)[i] = o;
    }
  } else {
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
      const float o = (srow[i] - mean) * rstd * g[i] + b[i];
      if (out_bf16) reinterpret_cast<__nv_bfloat16*>(out)[orow + i] = __float2bfloat16_rn(o);
      else reinterpret_cast<float*>(out)[orow + i] = o;
    }
  }
}

// ------------------------------------------------------------------------------------------
// GEGLU (attention.py:40-43): x, gate = chunk(2); gelu(gate) * x
// ------------------------------------------------------------------------------------------
__global__ void geglu_kernel(const float* __restrict__ h, float* __restrict__ out, int64_t rows, int inner) {
  pdl_prologue();
  const int64_t total = rows * inner;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / inner;
    const int j = (int)(i - r * inner);
    const float val = h[r * 2 * inner + j];
    const float gate = h[r * 2 * inner + inner + j];
    out[i] = gelu_erf(gate) * val;
  }
}

// ------------------------------------------------------------------------------------------
// token + position embedding and gradient-shrink forward value (phenaki_pytorch.py:194-199)
// ------------------------------------------------------------------------------------------
__global__ void token_embed_kernel(const int64_t* __restrict__ ids, const float* __restrict__ tok,
                                   const float* __restrict__ pos, float* __restrict__ out, int n, int dim,
                                   float alpha, float one_minus_alpha, int shrink, int64_t id_rows, int vocab_rows) {
  pdl_prologue();
  const int64_t row = blockIdx.x;
  const int p = (int)(row % n);
  int64_t id = ids[row % id_rows];  // the CFG null half replays the same ids
  // an id outside the table is a caller error (nn.Embedding raises; the Python entry points check); here it must at
  // least never read outside the table
  id = id < 0 ? 0 : (id >= vocab_rows ? vocab_rows - 1 : id);
  const float* t = tok + id * dim;
  const float* pe = pos + (int64_t)p * dim;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) {
    float x = __fadd_rn(pe[i], t[i]);  // pos_emb(arange) + token_emb(x)
    if (shrink) x = __fadd_rn(__fmul_rn(x, alpha), __fmul_rn(x, one_minus_alpha));
    out[row * dim + i] = x;
  }
}

// Persistent variant for p2 % 4 == 0 and K <= NJ * 1024: each thread owns the same NJ float4 positions of every token, so
// its gather offsets are computed once, gamma / beta (2 x 24 KB per token at K = 6144 -- twice the video bytes when
// every CTA re-reads them from L2) are staged once per CTA in shared memory, and the token itself stays in registers
// between the two LayerNorm passes.  ~60 registers -> 4 CTAs per SM keep ~96 KB of video loads in flight per SM.
template <int NJ>
__global__ void __launch_bounds__(256, 4) patchify_ln_reg_kernel(const float* __restrict__ video, int C, int F, int H,
                                                                 int W, int f0, int nt, int pt, int p1, int p2,
                                                                 const float* __restrict__ g, const float* __restrict__ b,
                                                                 void* __restrict__ out, int out_bf16, int tokens) {
  pdl_trigger();
  extern __shared__ float4 sgb[];  // [K4] gamma, [K4] beta
  __shared__ float red[32];
  const int hh = H / p1, ww = W / p2;
  const int K = C * pt * p1 * p2, K4 = K >> 2;
  const int plane = H * W;
  const int runs = p2 >> 2;
  int off[NJ];  // float offset of this thread's j-th float4 inside the token's (c, dt, dy, dx) gather; -1: none
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int i = threadIdx.x + 256 * j;
    off[j] = -1;
    if (i < K4) {
      const int dx4 = i % runs;
      int r = i / runs;  // (c, dt, dy)
      const int dy = r % p1; r /= p1;
      const int dt = r % pt;
      const int c = r / pt;
      off[j] = (c * F + dt) * plane + dy * W + dx4 * 4;
      sgb[i] = __ldg(reinterpret_cast<const float4*>(g) + i);
      sgb[K4 + i] = __ldg(reinterpret_cast<const float4*>(b) + i);
    }
  }
  pdl_wait();  // gamma / beta are weights; the video may come from the previous kernel (decode -> encode chains)
  for (int token = blockIdx.x; token < tokens; token += gridDim.x) {
    int tok = token;
    const int wi = tok % ww; tok /= ww;
    const int hi = tok % hh; tok /= hh;
    const int ti = tok % nt;
    const int bi = tok / nt;
    const float* base = video + ((int64_t)bi * C * F + f0 + (int64_t)ti * pt) * plane + (int64_t)hi * p1 * W + wi * p2;
    float4 v[NJ];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (off[j] >= 0) v[j] = __ldg(reinterpret_cast<const float4*>(base + off[j]));
    }
#pragma unroll
    for (int j = 0; j < NJ; ++j) s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
    const float mean = block_sum(s, red) / (float)K;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j)
      if (off[j] >= 0) {
        const float a = v[j].x - mean, bq = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
        q += (a * a + bq * bq) + (c * c + d * d);
      }
    const float rstd = rsqrtf(block_sum(q, red) / (float)K + 1e-5f);
    const int64_t orow = (int64_t)token * K;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if (off[j] < 0) continue;
      const int i = threadIdx.x + 256 * j;
      const float4 gg = sgb[i], bb = sgb[K4 + i];
      float4 o;
      o.x = (v[j].x - mean) * rstd * gg.x + bb.x;
      o.y = (v[j].y - mean) * rstd * gg.y + bb.y;
      o.z = (v[j].z - mean) * rstd * gg.z + bb.z;
      o.w = (v[j].w - mean) * rstd * gg.w + bb.w;
      if (out_bf16)
        reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + orow)[i] =
            make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
      else
        reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + orow)[i] = o;
    }
  }
}

// ------------------------------------------------------------------------------------------
// LFQ ids (oracle/lfq.py; call site cvivit.py:570).  Warp per row.
// ------------------------------------------------------------------------------------------
template <int XPL /* x values per lane = dim / 32 */>
__global__ void __launch_bounds__(256) lfq_kernel(const float* __restrict__ x, const float* __restrict__ wp,
                                                  const float* __restrict__ bp, int64_t* __restrict__ ids,
                                                  float* __restrict__ proj, int64_t rows, int dim, int bits) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * dim;
  int64_t id = 0;
  if (XPL > 0) {
    // the token row stays in registers; all `bits` dot products advance together (independent FMA chains)
    float xv[XPL > 0 ? XPL : 1];
#pragma unroll
    for (int i = 0; i < XPL; ++i) xv[i] = xr[lane + 32 * i];
    for (int d0 = 0; d0 < bits; d0 += 8) {
      float acc[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
      for (int i = 0; i < XPL; ++i)
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (d0 + e < bits) acc[e] = fmaf(xv[i], __ldg(wp + (int64_t)(d0 + e) * dim + lane + 32 * i), acc[e]);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (d0 + e >= bits) break;
        const float a = warp_sum(acc[e]) + bp[d0 + e];
        if (proj && lane == 0) proj[row * bits + d0 + e] = a;
        if (a > 0.f) id |= (int64_t)1 << (bits - 1 - d0 - e);
      }
    }
  } else {
    for (int d = 0; d < bits; ++d) {
      const float* w = wp + (int64_t)d * dim;
      float acc = 0.f;
      for (int i = lane; i < dim; i += 32) acc = fmaf(xr[i], __ldg(w + i), acc);
      acc = warp_sum(acc) + bp[d];
      if (proj && lane == 0) proj[row * bits + d] = acc;
      if (acc > 0.f) id |= (int64_t)1 << (bits - 1 - d);
    }
  }
  if (lane == 0) ids[row] = id;
}

// ------------------------------------------------------------------------------------------
// norm_out LayerNorm of the temporal transformer (attention.py:308,332) fused with the LFQ projection and sign
// quantisation (cvivit.py:570): the normalised row never leaves registers.  project_in's [bits, dim] weight is
// staged once per CTA in shared memory (32 KB at dim 512); each warp normalises R rows and advances all
// bits x R dot products together, so every 16-B weight read from shared memory feeds R FMAs x 4.
// ------------------------------------------------------------------------------------------
template <int VEC /* float4 per lane = dim / 128 */, int R /* rows per warp */>
__global__ void __launch_bounds__(256) ln_lfq_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                     const float* __restrict__ b, const float* __restrict__ wp,
                                                     const float* __restrict__ bp, int64_t* __restrict__ ids,
                                                     float* __restrict__ out_norm, float* __restrict__ proj,
                                                     int64_t rows, int dim, int bits) {
  constexpr int MAXB = 16;
  extern __shared__ float4 swp[];  // [bits][dim / 4]
  pdl_trigger();
  const int d4 = dim >> 2;
  for (int i = threadIdx.x; i < bits * d4; i += blockDim.x) swp[i] = __ldg(reinterpret_cast<const float4*>(wp) + i);
  pdl_wait();  // the weights above are not produced by the previous kernel; x is
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t row0 = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * R;
  if (row0 >= rows) return;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  const float4* b4 = reinterpret_cast<const float4*>(b);
  float4 y[R][VEC];
#pragma unroll
  for (int rr = 0; rr < R; ++rr) {
    const int64_t row = row0 + rr < rows ? row0 + rr : rows - 1;  // tail rows recompute the last row (not stored)
    const float4* xr = reinterpret_cast<const float4*>(x + row * dim);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      y[rr][j] = xr[lane + 32 * j];
      s += (y[rr][j].x + y[rr][j].y) + (y[rr][j].z + y[rr][j].w);
    }
    const float mean = warp_sum(s) / (float)dim;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float a = y[rr][j].x - mean, bb = y[rr][j].y - mean, c = y[rr][j].z - mean, d = y[rr][j].w - mean;
      q += (a * a + bb * bb) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)dim + 1e-5f);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float4 gg = g4[lane + 32 * j], bb = b4[lane + 32 * j];
      y[rr][j].x = (y[rr][j].x - mean) * rstd * gg.x + bb.x;
      y[rr][j].y = (y[rr][j].y - mean) * rstd * gg.y + bb.y;
      y[rr][j].z = (y[rr][j].z - mean) * rstd * gg.z + bb.z;
      y[rr][j].w = (y[rr][j].w - mean) * rstd * gg.w + bb.w;
      if (out_norm && row0 + rr < rows) reinterpret_cast<float4*>(out_norm + row * dim)[lane + 32 * j] = y[rr][j];
    }
  }
  float acc[R][MAXB];
#pragma unroll
  for (int rr = 0; rr < R; ++rr)
#pragma unroll
    for (int e = 0; e < MAXB; ++e) acc[rr][e] = 0.f;
#pragma unroll
  for (int e = 0; e < MAXB; ++e) {
    if (e < bits) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float4 w = swp[e * d4 + lane + 32 * j];
#pragma unroll
        for (int rr = 0; rr < R; ++rr)
          acc[rr][e] = fmaf(y[rr][j].x, w.x, fmaf(y[rr][j].y, w.y, fmaf(y[rr][j].z, w.z, fmaf(y[rr][j].w, w.w, acc[rr][e]))));
      }
    }
  }
#pragma unroll
  for (int rr = 0; rr < R; ++rr) {
    int64_t id = 0;
#pragma unroll
    for (int e = 0; e < MAXB; ++e) {
      if (e < bits) {
        const float a = warp_sum(acc[rr][e]) + __ldg(bp + e);
        if (proj && lane == 0 && row0 + rr < rows) proj[(row0 + rr) * bits + e] = a;
        if (a > 0.f) id |= (int64_t)1 << (bits - 1 - e);
      }
    }
    if (lane == 0 && row0 + rr < rows) ids[row0 + rr] = id;
  }
}

// ------------------------------------------------------------------------------------------
// PEG depthwise 3x3x3 conv + bias + residual (attention.py:64-85, caller :323).
// w is tap-major [27][D] (packed by the host module from dsconv.weight[D,1,3,3,3]).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t peg_phys_row(int64_t r_log, int T, int HW, int layout) {
  if (layout == 0) return r_log;
  // reference buffer is '(b h w) t d' reinterpreted as (b,t,h,w,d); ours is stored (b,t,h,w)
  const int64_t s = r_log / T;
  const int tau = (int)(r_log - s * T);
  const int64_t b2 = s / HW;
  const int hw = (int)(s - b2 * HW);
  return (b2 * T + tau) * HW + hw;
}

__global__ void __launch_bounds__(128) peg_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                  const float* __restrict__ bias, float* __restrict__ y, int T, int H,
                                                  int W, int D, int pad_t0, int layout) {
  pdl_prologue();
  // one CTA per logical position; the 27 neighbour rows are resolved once (the index maps need divisions),
  // then every thread streams float4 channels: x rows and the tap-major weights are read fully coalesced.
  __shared__ int s_src[27];
  __shared__ int s_out;
  const int r_log = blockIdx.x;
  const int HW = H * W;
  if (threadIdx.x < 27) {
    int rem = r_log % (T * HW);
    const int bi = r_log / (T * HW);
    const int t = rem / HW; rem -= t * HW;
    const int h = rem / W;
    const int wq = rem - h * W;
    const int kt = threadIdx.x / 9, kh = (threadIdx.x / 3) % 3, kw = threadIdx.x % 3;
    const int ts = t + kt - pad_t0, hs = h + kh - 1, ws = wq + kw - 1;
    int src = -1;
    if (ts >= 0 && ts < T && hs >= 0 && hs < H && ws >= 0 && ws < W)
      src = (int)peg_phys_row(((int64_t)(bi * T + ts) * H + hs) * W + ws, T, HW, layout);
    s_src[threadIdx.x] = src;
    if (threadIdx.x == 0) s_out = (int)peg_phys_row(r_log, T, HW, layout);
  }
  __syncthreads();
  const int64_t out_row = s_out;
  for (int d4 = threadIdx.x; d4 < (D >> 2); d4 += blockDim.x) {
    float4 acc = __ldg(reinterpret_cast<const float4*>(bias) + d4);
#pragma unroll
    for (int tap = 0; tap < 27; ++tap) {
      const int src = s_src[tap];
      if (src < 0) continue;
      const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (int64_t)src * D) + d4);
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w + (int64_t)tap * D) + d4);
      acc.x = fmaf(xv.x, wv.x, acc.x);
      acc.y = fmaf(xv.y, wv.y, acc.y);
      acc.z = fmaf(xv.z, wv.z, acc.z);
      acc.w = fmaf(xv.w, wv.w, acc.w);
    }
    const float4 xs = __ldg(reinterpret_cast<const float4*>(x + out_row * D) + d4);
    reinterpret_cast<float4*>(y + out_row * D)[d4] = make_float4(acc.x + xs.x, acc.y + xs.y, acc.z + xs.z, acc.w + xs.w);
  }
}

// Frame-tiled variant: one CTA per (logical frame (b,t), 64-channel chunk).  The (up to) three temporal slices the
// 3x3x3 stencil touches are staged once in shared memory (3 x H*W x 64 floats) together with the 27 x 64 taps, so
// every x row is fetched 3 times from L2 instead of 27.  Each thread owns a channel quad and one image ROW: for every
// (kt, kh) it pulls the W (+2 halo) neighbours of that row into registers once and applies the three kw taps to all W
// outputs -- ~1/4 of the issue slots of a tap-by-tap loop.  Used when the frame fits (H*W <= 128) and W is 4, 8 or 16.
constexpr int PEG_CH = 64;
template <int WW>
__global__ void __launch_bounds__(256) peg_tiled_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ y, int T,
                                                        int H, int D, int pad_t0, int layout) {
  pdl_prologue();
  extern __shared__ float peg_smem[];
  const int P = H * WW;
  float4* s_x = reinterpret_cast<float4*>(peg_smem);                  // [3][P][16] channel quads
  float4* s_w = s_x + 3 * P * (PEG_CH / 4);                           // [27][16]
  int* s_row = reinterpret_cast<int*>(s_w + 27 * (PEG_CH / 4));       // [3][P] physical rows (-1: outside the clip)
  const int frame = blockIdx.x, ch0 = blockIdx.y * PEG_CH;
  const int t = frame % T, bi = frame / T;
  const int nthr = blockDim.x;
  for (int i = threadIdx.x; i < 3 * P; i += nthr) {
    const int kt = i / P, pp = i - kt * P;
    const int ts = t + kt - pad_t0;
    s_row[i] = (ts >= 0 && ts < T) ? (int)peg_phys_row(((int64_t)bi * T + ts) * P + pp, T, P, layout) : -1;
  }
  for (int i = threadIdx.x; i < 27 * (PEG_CH / 4); i += nthr)
    s_w[i] = __ldg(reinterpret_cast<const float4*>(w + (int64_t)(i / (PEG_CH / 4)) * D + ch0) + (i % (PEG_CH / 4)));
  __syncthreads();
  const int total = 3 * P * (PEG_CH / 4);
  for (int i0 = threadIdx.x; i0 < total; i0 += 8 * nthr) {  // 8 independent 16-byte loads in flight per thread
    float4 v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = i0 + u * nthr;
      v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < total) {
        const int r = s_row[i / (PEG_CH / 4)];
        if (r >= 0) v[u] = __ldg(reinterpret_cast<const float4*>(x + (int64_t)r * D + ch0) + (i % (PEG_CH / 4)));
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) if (i0 + u * nthr < total) s_x[i0 + u * nthr] = v[u];
  }
  __syncthreads();
  const int c4 = threadIdx.x & 15, h = threadIdx.x >> 4;  // 16 channel quads x H rows
  if (h >= H) return;
  const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + ch0) + c4);
  float4 acc[WW];
#pragma unroll
  for (int i = 0; i < WW; ++i) acc[i] = bv;
#pragma unroll
  for (int kt = 0; kt < 3; ++kt) {
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hs = h + kh - 1;
      if (hs < 0 || hs >= H) continue;
      float4 xr[WW + 2];
      xr[0] = make_float4(0.f, 0.f, 0.f, 0.f);
      xr[WW + 1] = xr[0];
      const float4* src = s_x + (kt * P + hs * WW) * (PEG_CH / 4) + c4;
#pragma unroll
      for (int i = 0; i < WW; ++i) xr[i + 1] = src[i * (PEG_CH / 4)];
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const float4 wv = s_w[((kt * 3 + kh) * 3 + kw) * (PEG_CH / 4) + c4];
#pragma unroll
        for (int i = 0; i < WW; ++i) {
          acc[i].x = fmaf(xr[i + kw].x, wv.x, acc[i].x);
          acc[i].y = fmaf(xr[i + kw].y, wv.y, acc[i].y);
          acc[i].z = fmaf(xr[i + kw].z, wv.z, acc[i].z);
          acc[i].w = fmaf(xr[i + kw].w, wv.w, acc[i].w);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < WW; ++i) {
    const int pp = h * WW + i;
    const float4 xs = s_x[(pad_t0 * P + pp) * (PEG_CH / 4) + c4];  // residual: slice ts == t
    const int orow = s_row[pad_t0 * P + pp];
    reinterpret_cast<float4*>(y + (int64_t)orow * D + ch0)[c4] =
        make_float4(acc[i].x + xs.x, acc[i].y + xs.y, acc[i].z + xs.z, acc[i].w + xs.w);
  }
}

template <int WW>
static int launch_peg_tiled(const float* x, const float* w, const float* b, float* y, int B, int T, int H, int D,
                            int pad_t0, int layout, cudaStream_t st) {
  const int P = H * WW;
  const size_t smem = (size_t)(3 * P * PEG_CH + 27 * PEG_CH) * sizeof(float) + (size_t)3 * P * sizeof(int);
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(peg_tiled_kernel<WW>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)((3 * 128 * PEG_CH + 27 * PEG_CH) * sizeof(float) + 3 * 128 * sizeof(int))));
    mark_configured(&configured_mask);
  }
  PHK_CUDA(launch_pdl(peg_tiled_kernel<WW>, dim3((unsigned)(B * T), (unsigned)(D / PEG_CH)), dim3((unsigned)(16 * H)), smem,
                      st, x, w, b, y, T, H, D, pad_t0, layout));
  return 0;
}

// ------------------------------------------------------------------------------------------
// ContinuousPositionBias (attention.py:257-275).  Weight-only: MLP over distinct deltas
// (table kernel), then expansion to (heads, n, n).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cpb_table_kernel(phk_cpb_t c, int d0, int d1, int d2,
                                                        float* __restrict__ table) {
  pdl_prologue();
  extern __shared__ float sm[];
  float* h1 = sm;
  float* h2 = sm + c.hidden;
  const int u = blockIdx.x;
  const int s1 = 2 * d1 - 1, s2 = 2 * d2 - 1;
  int delta[3];
  delta[0] = u / (s1 * s2) - (d0 - 1);
  delta[1] = (u / s2) % s1 - (d1 - 1);
  delta[2] = u % s2 - (d2 - 1);
  float in[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int a = delta[i] < 0 ? -delta[i] : delta[i];
    const float sg = delta[i] > 0 ? 1.f : (delta[i] < 0 ? -1.f : 0.f);
    in[i] = sg * logf((float)(a + 1));  // sign(rel) * log(|rel| + 1)   (attention.py:266)
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int j = threadIdx.x; j < c.hidden; j += blockDim.x) {
    float a = c.b0[j];
    for (int i = 0; i < c.num_dims; ++i) a = fmaf(in[i], c.w0[j * c.num_dims + i], a);
    h1[j] = a > 0.f ? a : 0.1f * a;
  }
  __syncthreads();
  for (int j = wid; j < c.hidden; j += nw) {
    float a = 0.f;
    for (int k = lane; k < c.hidden; k += 32) a = fmaf(h1[k], c.w1[(int64_t)j * c.hidden + k], a);
    a = warp_sum(a) + c.b1[j];
    if (lane == 0) h2[j] = a > 0.f ? a : 0.1f * a;
  }
  __syncthreads();
  for (int j = wid; j < c.heads; j += nw) {
    float a = 0.f;
    for (int k = lane; k < c.hidden; k += 32) a = fmaf(h2[k], c.w2[(int64_t)j * c.hidden + k], a);
    a = warp_sum(a) + c.b2[j];
    if (lane == 0) table[(int64_t)u * c.heads + j] = a;
  }
}

__global__ void cpb_expand_kernel(const float* __restrict__ table, float* __restrict__ out, int heads, int d0,
                                  int d1, int d2) {
  pdl_prologue();
  const int n = d0 * d1 * d2;
  const int64_t total = (int64_t)n * n;
  const int s1 = 2 * d1 - 1, s2 = 2 * d2 - 1;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / n), j = (int)(idx % n);
    const int i0 = i / (d1 * d2), i1 = (i / d2) % d1, i2 = i % d2;
    const int j0 = j / (d1 * d2), j1 = (j / d2) % d1, j2 = j % d2;
    const int u = ((i0 - j0 + d0 - 1) * s1 + (i1 - j1 + d1 - 1)) * s2 + (i2 - j2 + d2 - 1);
    for (int h = 0; h < heads; ++h) out[(int64_t)h * total + idx] = table[(int64_t)u * heads + h];
  }
}

// ------------------------------------------------------------------------------------------
// CFG + gumbel argmax + confidence (phenaki_pytorch.py:161, 83-93, 506-509, 547-550).
// One CTA per token row, single pass over the V logits: running (argmax of perturbed logit,
// max / sum-exp of the guided logit).  fp32 op sequence mirrors the eager reference
// (sub, mul, add, div, add -- no FMA contraction) so argmax decisions agree bit for bit
// whenever logf agrees.
// ------------------------------------------------------------------------------------------
struct ArgBest { float y; int idx; };
__device__ __forceinline__ ArgBest better(ArgBest a, ArgBest b) {
  // larger y wins; ties -> lower index (torch.argmax returns the first maximal index)
  if (b.y > a.y || (b.y == a.y && b.idx < a.idx)) return b;
  return a;
}

__global__ void __launch_bounds__(512) sample_tokens_kernel(const float* __restrict__ cond,
                                                            const float* __restrict__ nul, int64_t ld,
                                                            const float* __restrict__ u, uint64_t seed,
                                                            uint64_t offset, float cond_scale, float temperature,
                                                            const uint8_t* __restrict__ mask,
                                                            int64_t* __restrict__ ids, int64_t* __restrict__ pred_out,
                                                            float* __restrict__ score_out, int V, int64_t seg_len,
                                                            int64_t seg_stride, int64_t seg_off) {
  pdl_prologue();
  __shared__ float s_y[16], s_m[16], s_s[16];
  __shared__ int s_i[16];
  const int64_t row = blockIdx.x;
  // logits[:, prime_len:] (phenaki_pytorch.py:503-504): token row -> row of the (b, prime+n) logits
  const int64_t lrow = seg_len > 0 ? (row / seg_len) * seg_stride + seg_off + row % seg_len : row;
  const float* cr = cond + lrow * ld;
  const float* nr = nul ? nul + lrow * ld : nullptr;
  const float* ur = u ? u + row * (int64_t)V : nullptr;
  const float T = fmaxf(temperature, 1e-10f);
  const float inv_T = 1.0f / T;
  ArgBest best{-FLT_MAX, 0x7fffffff};
  float m = -FLT_MAX, ssum = 0.f;
  for (int v0 = threadIdx.x * 4; v0 < V; v0 += blockDim.x * 4) {
    float uu[4], gg[4];
    if (ur) {
#pragma unroll
      for (int j = 0; j < 4; ++j) uu[j] = (v0 + j < V) ? ur[v0 + j] : 0.5f;
    } else {
      // statistical mode: in-kernel Philox noise, the same counters and gumbel transform as the fused logits head
      const uint64_t ctr = offset + (uint64_t)row * (uint64_t)((V + 3) / 4) + (uint64_t)(v0 >> 2);
      uint32_t r[4];
      philox4x32<kNoiseRounds>((uint32_t)ctr, (uint32_t)(ctr >> 32), 0u, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), r);
#pragma unroll
      for (int j = 0; j < 4; ++j) gg[j] = gumbel_from_bits(r[j]);
    }
    if (!ur && v0 + 3 < V && ((ld & 3) == 0)) {
      // statistical mode (in-kernel noise): vectorised loads and fast intrinsics; not bit-comparable anyway
      const float4 c4 = *reinterpret_cast<const float4*>(cr + v0);
      float l4[4] = {c4.x, c4.y, c4.z, c4.w};
      if (nr) {
        const float4 n4 = *reinterpret_cast<const float4*>(nr + v0);
        const float nn[4] = {n4.x, n4.y, n4.z, n4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) l4[j] = fmaf(l4[j] - nn[j], cond_scale, nn[j]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float l = l4[j];
        const float y = fmaf(l, inv_T, gg[j]);
        if (y > best.y) { best.y = y; best.idx = v0 + j; }
        if (l > m) { ssum = ssum * __expf(m - l) + 1.f; m = l; } else { ssum += __expf(l - m); }
      }
      continue;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int v = v0 + j;
      if (v >= V) break;
      float l = cr[v];
      if (nr) { const float nn = nr[v]; l = __fadd_rn(nn, __fmul_rn(__fsub_rn(l, nn), cond_scale)); }
      // injected draws: the reference's op sequence (phenaki_pytorch.py:83-93); in-kernel noise: gumbel_from_bits
      const float g = ur ? -logf(__fadd_rn(-logf(__fadd_rn(uu[j], 1e-10f)), 1e-10f)) : gg[j];
      const float y = ur ? __fadd_rn(__fdiv_rn(l, T), g) : fmaf(l, inv_T, g);
      if (y > best.y) { best.y = y; best.idx = v; }
      if (l > m) { ssum = ssum * expf(m - l) + 1.f; m = l; } else { ssum += expf(l - m); }
    }
  }
  // block combine
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgBest ob{__shfl_xor_sync(0xffffffffu, best.y, o), __shfl_xor_sync(0xffffffffu, best.idx, o)};
    best = better(best, ob);
    const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, ssum, o);
    const float nm = fmaxf(m, om);
    ssum = ssum * expf(m - nm) + os * expf(om - nm);
    m = nm;
  }
  if (lane == 0) { s_y[wid] = best.y; s_i[wid] = best.idx; s_m[wid] = m; s_s[wid] = ssum; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < nw; ++w) {
      best = better(best, ArgBest{s_y[w], s_i[w]});
      const float nm = fmaxf(m, s_m[w]);
      ssum = ssum * expf(m - nm) + s_s[w] * expf(s_m[w] - nm);
      m = nm;
    }
    const int pred = best.idx;
    float l = cr[pred];
    if (nr) { const float nn = nr[pred]; l = __fadd_rn(nn, __fmul_rn(__fsub_rn(l, nn), cond_scale)); }
    const float p = expf(l - m) / ssum;
    const bool mk = mask ? mask[row] != 0 : true;
    if (pred_out) pred_out[row] = pred;
    if (ids && mk) ids[row] = pred;                                   // where(mask, pred, ids)   (:509)
    if (score_out) score_out[row] = mk ? (1.0f - p) : -1e4f;          // (:547-550)
  }
}

// ------------------------------------------------------------------------------------------
// Cosine-schedule re-masking (phenaki_pytorch.py:485-491).  Rank by counting: element i is in
// the top-k iff fewer than k elements beat it (greater score, or equal score and lower index).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) topk_mask_kernel(const float* __restrict__ scores, int n, int k,
                                                         uint8_t* __restrict__ mask, int64_t* __restrict__ ids,
                                                         int64_t mask_id) {
  pdl_prologue();
  extern __shared__ float sc[];
  const int64_t row = blockIdx.x;
  for (int i = threadIdx.x; i < n; i += blockDim.x) sc[i] = scores[row * n + i];
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float si = sc[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const float sj = sc[j];
      rank += (sj > si) || (sj == si && j < i);
    }
    const uint8_t mk = rank < k;
    mask[row * n + i] = mk;
    if (mk) ids[row * n + i] = mask_id;                               // where(mask, mask_id, ids)  (:491)
  }
}

// ------------------------------------------------------------------------------------------
// Critic head + CFG + annealed noise (phenaki_pytorch.py:246-249, 263, 544-545).  Warp per row.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) critic_scores_kernel(const float* __restrict__ xc, const float* __restrict__ xn,
                                                            const float* __restrict__ w, const float* __restrict__ b,
                                                            const float* __restrict__ u, float cond_scale,
                                                            float noise_K, float noise_mult, float* __restrict__ out,
                                                            int64_t rows, int dim, int64_t seg_len, int64_t seg_stride,
                                                            int64_t seg_off) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int64_t xrow = seg_len > 0 ? (row / seg_len) * seg_stride + seg_off + row % seg_len : row;  // scores[:, prime:] (:528-529)
  float a = 0.f, c = 0.f;
  for (int i = lane; i < dim; i += 32) {
    const float wi = __ldg(w + i);
    a = fmaf(xc[xrow * dim + i], wi, a);
    if (xn) c = fmaf(xn[xrow * dim + i], wi, c);
  }
  a = warp_sum(a) + b[0];
  float sc = a;
  if (xn) { c = warp_sum(c) + b[0]; sc = __fadd_rn(c, __fmul_rn(__fsub_rn(a, c), cond_scale)); }
  if (u) sc = __fadd_rn(sc, __fmul_rn(__fmul_rn(noise_K, __fsub_rn(u[row], 0.5f)), noise_mult));
  if (lane == 0) out[row] = sc;
}

// null + (cond - null) * scale  (phenaki_pytorch.py:161), eager op order (sub, mul, add)
__global__ void cfg_combine_kernel(const float* __restrict__ cond, const float* __restrict__ nul, float scale,
                                   float* __restrict__ out, int64_t n) {
  pdl_prologue();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float nn = nul[i];
    out[i] = __fadd_rn(nn, __fmul_rn(__fsub_rn(cond[i], nn), scale));
  }
}


// ------------------------------------------------------------------------------------------
// LFQ indices_to_codes + project_out (cvivit.py:437-439; vector-quantize-pytorch LFQ.indices_to_codes):
// bit j (MSB first) of the id selects +1 / -1, then Linear(bits, dim).  One thread per output element; the
// [dim, bits] weight (32 KB at dim 512) stays in L1.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) lfq_codes_kernel(const int64_t* __restrict__ ids, const float* __restrict__ w,
                                                        const float* __restrict__ b, float* __restrict__ out,
                                                        int64_t rows, int dim, int bits) {
  pdl_prologue();
  const int64_t total = rows * dim;
  const bool vec = (bits % 4 == 0) && ((reinterpret_cast<uintptr_t>(w) & 15) == 0);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / dim;
    const int d = (int)(i - r * dim);
    const int64_t id = ids[r];
    const float* wr = w + (int64_t)d * bits;
    float acc = 0.f;
    if (vec) {  // the weight row of this output (bits floats, 64 B at 16 bits) as 16-byte loads, all issued up front
      for (int j = 0; j < bits; j += 4) {
        const float4 wv = __ldg(reinterpret_cast<const float4*>(wr + j));
        acc += ((id >> (bits - 1 - j)) & 1) ? wv.x : -wv.x;
        acc += ((id >> (bits - 2 - j)) & 1) ? wv.y : -wv.y;
        acc += ((id >> (bits - 3 - j)) & 1) ? wv.z : -wv.z;
        acc += ((id >> (bits - 4 - j)) & 1) ? wv.w : -wv.w;
      }
    } else {
      for (int j = 0; j < bits; ++j) {
        const float wv = __ldg(wr + j);
        acc += ((id >> (bits - 1 - j)) & 1) ? wv : -wv;
      }
    }
    out[i] = acc + __ldg(b + d);
  }
}

// ------------------------------------------------------------------------------------------
// Un-patchify (cvivit.py:286-295: Rearrange 'b t h w (c pt p1 p2) -> b c (t pt) (h p1) (w p2)'), the mirror of
// patchify_ln: P [B*nt*hh*ww, C*pt*p1*p2] -> frames [f0, f0 + nt*pt) of video (B,C,F,H,W).  Threads walk the
// OUTPUT in memory order (coalesced stores); the matching reads are p2-float contiguous runs of one P row.
// ------------------------------------------------------------------------------------------
template <int V /* floats per thread: 4 or 1 */>
__global__ void __launch_bounds__(256) unpatchify_kernel(const float* __restrict__ P, int64_t ldp,
                                                         float* __restrict__ video, int B, int C, int F, int H,
                                                         int W, int f0, int nt, int pt, int p1, int p2) {
  pdl_prologue();
  const int hh = H / p1, ww = W / p2, Wv = W / V;
  const int64_t total = (int64_t)B * C * nt * pt * H * Wv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int xv = (int)(r % Wv); r /= Wv;
    const int y = (int)(r % H); r /= H;
    const int f = (int)(r % (nt * pt)); r /= (nt * pt);
    const int c = (int)(r % C);
    const int b = (int)(r / C);
    const int x = xv * V;
    const int ti = f / pt, dt = f - ti * pt, hi = y / p1, dy = y - hi * p1, wi = x / p2, dx = x - wi * p2;
    const int64_t row = (((int64_t)b * nt + ti) * hh + hi) * ww + wi;
    const int64_t col = (((int64_t)c * pt + dt) * p1 + dy) * p2 + dx;
    float* dst = video + ((((int64_t)b * C + c) * F + f0 + f) * H + y) * W + x;
    if (V == 4) *reinterpret_cast<float4*>(dst) = *reinterpret_cast<const float4*>(P + row * ldp + col);
    else *dst = P[row * ldp + col];
  }
}
}  // namespace phk

// ==========================================================================================
// C ABI
// ==========================================================================================
using namespace phk;

extern "C" int phk_layernorm(const float* x, const float* gamma, const float* beta, void* out, void* raw_bf16,
                             int64_t rows, int32_t dim, int32_t out_bf16, int64_t seg_len, int64_t seg_stride,
                             int64_t seg_off, phk_stream_t s) {
  Prof prof_(FAM_LAYERNORM, s, (double)rows * dim * 8.0);
  PHK_REQUIRE(x && gamma && beta && out, PHK_E_ARG, "phk_layernorm: null pointer");
  PHK_REQUIRE(rows >= 0 && dim > 0, PHK_E_ARG, "phk_layernorm: bad size");
  if (rows == 0) return 0;
  cudaStream_t st = to_stream(s);
  __nv_bfloat16* raw = reinterpret_cast<__nv_bfloat16*>(raw_bf16);
  if (dim % 128 == 0 && dim <= 1024) {
    const int wpb = 8;
    const unsigned grid = (unsigned)((rows + wpb - 1) / wpb);
    switch (dim / 128) {
      case 1: PHK_CUDA(launch_pdl(ln_warp_kernel<1>, dim3(grid), dim3(256), (size_t)(0), st, x, gamma, beta, out, raw, rows, dim, out_bf16, seg_len, seg_stride, seg_off)); break;
      case 2: PHK_CUDA(launch_pdl(ln_warp_kernel<2>, dim3(grid), dim3(256), (size_t)(0), st, x, gamma, beta, out, raw, rows, dim, out_bf16, seg_len, seg_stride, seg_off)); break;
      case 3: PHK_CUDA(launch_pdl(ln_warp_kernel<3>, dim3(grid), dim3(256), (size_t)(0), st, x, gamma, beta, out, raw, rows, dim, out_bf16, seg_len, seg_stride, seg_off)); break;
      case 4: PHK_CUDA(launch_pdl(ln_warp_kernel<4>, dim3(grid), dim3(256), (size_t)(0), st, x, gamma, beta, out, raw, rows, dim, out_bf16, seg_len, seg_stride, seg_off)); break;
      case 5: PHK_CUDA(launch_pdl(ln_warp_kernel<5>, dim3(grid), dim3(256), (size_t)(0), st, x, gamma, beta, out, raw, rows, dim, out_bf16, seg_len, seg_stride, seg_off)); break;
      case 6: PHK_CUDA(launch_pdl(ln_warp_kernel<6>, dim3(grid), dim3(256), (size_t)(0), st, x, gamma, beta, out, raw, rows, dim, out_bf16, seg_len, seg_stride, seg_off)); break;
      case 7: PHK_CUDA(launch_pdl(ln_warp_kernel<7>, dim3(grid), dim3(256), (size_t)(0), st, x, gamma, beta, out, raw, rows, dim, out_bf16, seg_len, seg_stride, seg_off)); break;
      default: PHK_CUDA(launch_pdl(ln_warp_kernel<8>, dim3(grid), dim3(256), (size_t)(0), st, x, gamma, beta, out, raw, rows, dim, out_bf16, seg_len, seg_stride, seg_off)); break;
    }
  } else {
    PHK_REQUIRE(dim <= 12288, PHK_E_UNSUPPORTED, "phk_layernorm: dim > 12288");
    PHK_CUDA(launch_pdl(ln_block_kernel, dim3((unsigned)rows), dim3(256), (size_t)(dim * sizeof(float)), st, x, gamma, beta, out, raw, dim, out_bf16, seg_len, seg_stride, seg_off));
  }
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_patchify_ln(const float* video, int32_t B, int32_t C, int32_t F, int32_t H, int32_t W, int32_t f0,
                               int32_t nt, int32_t pt, int32_t p1, int32_t p2, const float* ln_g, const float* ln_b,
                               void* out, int32_t out_bf16, phk_stream_t s) {
  Prof prof_(FAM_PATCHIFY, s, (double)B * C * nt * pt * H * W * 8.0);
  PHK_REQUIRE(video && ln_g && ln_b && out, PHK_E_ARG, "phk_patchify_ln: null pointer");
  PHK_REQUIRE(B > 0 && C > 0 && F > 0 && H > 0 && W > 0 && pt > 0 && p1 > 0 && p2 > 0 && nt >= 0, PHK_E_ARG,
              "phk_patchify_ln: bad size");
  PHK_REQUIRE(H % p1 == 0 && W % p2 == 0, PHK_E_SHAPE, "image size must be divisible by patch size (cvivit.py:271)");
  PHK_REQUIRE(f0 >= 0 && f0 + nt * pt <= F, PHK_E_SHAPE, "frame range outside the video");
  if (nt == 0) return 0;
  const int K = C * pt * p1 * p2;
  PHK_REQUIRE(K <= 14336, PHK_E_UNSUPPORTED, "patch feature size > 14336 floats (56 KB smem row)");
  const unsigned grid = (unsigned)((int64_t)B * nt * (H / p1) * (W / p2));
  const size_t smem = (size_t)K * sizeof(float);
  const bool vec = (p2 % 4 == 0) && (W % 4 == 0) && ((reinterpret_cast<uintptr_t>(video) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
  {  // token gathered by the TMA unit, double-buffered per CTA (patchify_tma.cu); 1 = shape not eligible
    const int rc = patchify_ln_tma_launch(video, B, C, F, H, W, f0, nt, pt, p1, p2, ln_g, ln_b, out, out_bf16, to_stream(s));
    if (rc == 0) { PHK_LAUNCH_CHECK(); return 0; }
    if (rc != 1) return rc;
  }
  if (vec && K <= 6 * 1024 && ((reinterpret_cast<uintptr_t>(ln_g) | reinterpret_cast<uintptr_t>(ln_b)) & 15) == 0) {
    // persistent, register-resident variant (4 CTAs per SM; gamma / beta staged once per CTA: 2 * K * 4 bytes of smem)
    PHK_REQUIRE((int64_t)C * F * H * W < (1LL << 31), PHK_E_UNSUPPORTED, "phk_patchify_ln: one video exceeds 2^31 elements");
    const unsigned pgrid = grid < 4u * kNumSMs ? grid : 4u * kNumSMs;
    const size_t gsmem = (size_t)2 * K * sizeof(float);
    static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
    if (!configured) {
      PHK_CUDA(cudaFuncSetAttribute(patchify_ln_reg_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 49152));
      PHK_CUDA(cudaFuncSetAttribute(patchify_ln_reg_kernel<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, 49152));
      mark_configured(&configured_mask);
    }
    if (K <= 3 * 1024) PHK_CUDA(launch_pdl(patchify_ln_reg_kernel<3>, dim3(pgrid), dim3(256), gsmem, to_stream(s), video, C, F, H, W, f0, nt, pt, p1, p2, ln_g, ln_b, out, out_bf16, (int)grid));
    else PHK_CUDA(launch_pdl(patchify_ln_reg_kernel<6>, dim3(pgrid), dim3(256), gsmem, to_stream(s), video, C, F, H, W, f0, nt, pt, p1, p2, ln_g, ln_b, out, out_bf16, (int)grid));
    PHK_LAUNCH_CHECK();
    return 0;
  }
  if (smem > 48 * 1024) {
    PHK_CUDA(cudaFuncSetAttribute(patchify_ln_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 57344));
    PHK_CUDA(cudaFuncSetAttribute(patchify_ln_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 57344));
  }
  if (vec) PHK_CUDA(launch_pdl(patchify_ln_kernel<true>, dim3(grid), dim3(256), (size_t)(smem), to_stream(s), video, C, F, H, W, f0, nt, pt, p1, p2, ln_g, ln_b, out, out_bf16));
  else PHK_CUDA(launch_pdl(patchify_ln_kernel<false>, dim3(grid), dim3(256), (size_t)(smem), to_stream(s), video, C, F, H, W, f0, nt, pt, p1, p2, ln_g, ln_b, out, out_bf16));
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_geglu(const float* h, float* out, int64_t rows, int32_t inner, phk_stream_t s) {
  Prof prof_(FAM_GEGLU, s, (double)rows * inner * 12.0);
  PHK_REQUIRE(h && out, PHK_E_ARG, "phk_geglu: null pointer");
  PHK_REQUIRE(rows >= 0 && inner > 0, PHK_E_ARG, "phk_geglu: bad size");
  if (rows == 0) return 0;
  const int64_t total = rows * inner;
  const unsigned grid = (unsigned)((total + 255) / 256 < (int64_t)kNumSMs * 16 ? (total + 255) / 256 : kNumSMs * 16);
  PHK_CUDA(launch_pdl(geglu_kernel, dim3(grid), dim3(256), (size_t)(0), to_stream(s), h, out, rows, inner));
  PHK_LAUNCH_CHECK();
  return 0;
}

// PHK_PREC_BF16X3 operand split (see include/phk.h): one thread per 4 columns, 8-byte bf16x4 stores into three segments
__global__ void __launch_bounds__(256) split3_kernel(const float* __restrict__ x, int64_t ld, __nv_bfloat16* __restrict__ out,
                                                     int64_t rows, int K, int Kp, int weights) {
  pdl_prologue();
  const int q = Kp / 4;  // float4 groups per row (Kp % 8 == 0)
  const int64_t total = rows * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / q;
    const int c = (int)(i - r * q) * 4;
    float v[4];
    const float* xr = x + r * ld + c;
    if (c + 3 < K && (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
      const float4 t = *reinterpret_cast<const float4*>(xr);
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = (c + j < K) ? xr[j] : 0.f;
    }
    float hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      hi[j] = __bfloat162float(__float2bfloat16_rn(v[j]));
      lo[j] = v[j] - hi[j];  // exact in fp32
    }
    const uint2 H = make_uint2(pack_bf16x2(hi[0], hi[1]), pack_bf16x2(hi[2], hi[3]));
    const uint2 Lo = make_uint2(pack_bf16x2(lo[0], lo[1]), pack_bf16x2(lo[2], lo[3]));
    __nv_bfloat16* o = out + r * 3 * (int64_t)Kp + c;
    *reinterpret_cast<uint2*>(o) = H;
    *reinterpret_cast<uint2*>(o + Kp) = weights ? Lo : H;
    *reinterpret_cast<uint2*>(o + 2 * (int64_t)Kp) = weights ? H : Lo;
  }
}

extern "C" int phk_split3(const float* x, int64_t ld, void* out, int64_t rows, int32_t K, int32_t weights, phk_stream_t s) {
  Prof prof_(FAM_GEMM_BF16, s, 0.0);
  PHK_REQUIRE(x && out, PHK_E_ARG, "phk_split3: null pointer");
  PHK_REQUIRE(rows >= 0 && K > 0 && ld >= K, PHK_E_ARG, "phk_split3: bad size");
  PHK_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, PHK_E_ARG, "phk_split3: output must be 16-byte aligned");
  if (rows == 0) return 0;
  const int Kp = (K + 7) / 8 * 8;
  const int64_t total = rows * (Kp / 4);
  const int64_t want = (total + 255) / 256;
  const unsigned blocks = (unsigned)(want < 148 * 16 ? want : 148 * 16);
  PHK_CUDA(launch_pdl(split3_kernel, dim3(blocks), dim3(256), (size_t)0, to_stream(s), x, ld, (__nv_bfloat16*)out, rows, (int)K, Kp,
                      (int)weights));
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_token_embed(const int64_t* ids, const float* tok, const float* pos, float* out, int32_t b, int32_t n,
                               int32_t dim, int32_t vocab_rows, float alpha, int32_t replicas, phk_stream_t s) {
  Prof prof_(FAM_EMBED, s);
  PHK_REQUIRE(ids && tok && pos && out, PHK_E_ARG, "phk_token_embed: null pointer");
  PHK_REQUIRE(b > 0 && n > 0 && dim > 0 && vocab_rows > 0, PHK_E_ARG, "phk_token_embed: bad size");
  const int shrink = alpha >= 0.f;
  // (1 - alpha) is evaluated in double by the reference's Python and rounded to fp32 at the mul
  const float oma = (float)(1.0 - (double)alpha);
  if (replicas < 1) replicas = 1;
  PHK_CUDA(launch_pdl(token_embed_kernel, dim3((unsigned)(b * n * replicas)), dim3(128), (size_t)(0), to_stream(s), ids, tok, pos, out, n, dim, alpha, oma, shrink, (int64_t)b * n, vocab_rows));
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_lfq_ids(const float* x, const float* wp, const float* bp, int64_t* ids, float* proj_out,
                           int64_t rows, int32_t dim, int32_t bits, phk_stream_t s) {
  Prof prof_(FAM_LFQ, s);
  PHK_REQUIRE(x && wp && bp && ids, PHK_E_ARG, "phk_lfq_ids: null pointer");
  PHK_REQUIRE(rows >= 0 && dim > 0 && bits > 0 && bits <= 62, PHK_E_ARG, "phk_lfq_ids: bad size");
  if (rows == 0) return 0;
  const dim3 lg((unsigned)((rows + 7) / 8)), lb(256);
  if (dim == 512) PHK_CUDA(launch_pdl(lfq_kernel<16>, lg, lb, (size_t)0, to_stream(s), x, wp, bp, ids, proj_out, rows, dim, bits));
  else if (dim == 256) PHK_CUDA(launch_pdl(lfq_kernel<8>, lg, lb, (size_t)0, to_stream(s), x, wp, bp, ids, proj_out, rows, dim, bits));
  else if (dim == 1024) PHK_CUDA(launch_pdl(lfq_kernel<32>, lg, lb, (size_t)0, to_stream(s), x, wp, bp, ids, proj_out, rows, dim, bits));
  else PHK_CUDA(launch_pdl(lfq_kernel<0>, lg, lb, (size_t)0, to_stream(s), x, wp, bp, ids, proj_out, rows, dim, bits));
  PHK_LAUNCH_CHECK();
  return 0;
}

template <int VEC>
static int launch_ln_lfq(const float* x, const float* g, const float* b, const float* wp, const float* bp, int64_t* ids,
                         float* out_norm, float* proj, int64_t rows, int dim, int bits, cudaStream_t st) {
  constexpr int R = 2;
  const size_t smem = (size_t)bits * dim * sizeof(float);
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(ln_lfq_kernel<VEC, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 16 * 1024 * 4));
    mark_configured(&configured_mask);
  }
  const unsigned grid = (unsigned)((rows + 8 * R - 1) / (8 * R));
  PHK_CUDA(launch_pdl(ln_lfq_kernel<VEC, R>, dim3(grid), dim3(256), smem, st, x, g, b, wp, bp, ids, out_norm, proj, rows, dim, bits));
  return 0;
}

extern "C" int phk_layernorm_lfq(const float* x, const float* gamma, const float* beta, const float* wp,
                                 const float* bp, int64_t* ids, float* out_norm, float* proj_out, int64_t rows,
                                 int32_t dim, int32_t bits, phk_stream_t s) {
  PHK_REQUIRE(x && gamma && beta && wp && bp && ids, PHK_E_ARG, "phk_layernorm_lfq: null pointer");
  PHK_REQUIRE(rows >= 0 && dim > 0 && bits > 0 && bits <= 62, PHK_E_ARG, "phk_layernorm_lfq: bad size");
  if (rows == 0) return 0;
  const bool fused = dim % 128 == 0 && dim <= 1024 && bits <= 16 && (reinterpret_cast<uintptr_t>(wp) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  if (!fused) {  // general shapes: LayerNorm then the stand-alone LFQ kernel (out_norm doubles as the scratch row buffer)
    PHK_REQUIRE(out_norm, PHK_E_UNSUPPORTED, "phk_layernorm_lfq: this shape needs out_norm as scratch");
    PHK_TRY(phk_layernorm(x, gamma, beta, out_norm, nullptr, rows, dim, 0, 0, 0, 0, s));
    return phk_lfq_ids(out_norm, wp, bp, ids, proj_out, rows, dim, bits, s);
  }
  Prof prof_(FAM_LFQ, s, (double)rows * dim * 4.0);
  cudaStream_t st = to_stream(s);
  switch (dim / 128) {
    case 1: PHK_TRY(launch_ln_lfq<1>(x, gamma, beta, wp, bp, ids, out_norm, proj_out, rows, dim, bits, st)); break;
    case 2: PHK_TRY(launch_ln_lfq<2>(x, gamma, beta, wp, bp, ids, out_norm, proj_out, rows, dim, bits, st)); break;
    case 3: PHK_TRY(launch_ln_lfq<3>(x, gamma, beta, wp, bp, ids, out_norm, proj_out, rows, dim, bits, st)); break;
    case 4: PHK_TRY(launch_ln_lfq<4>(x, gamma, beta, wp, bp, ids, out_norm, proj_out, rows, dim, bits, st)); break;
    case 5: PHK_TRY(launch_ln_lfq<5>(x, gamma, beta, wp, bp, ids, out_norm, proj_out, rows, dim, bits, st)); break;
    case 6: PHK_TRY(launch_ln_lfq<6>(x, gamma, beta, wp, bp, ids, out_norm, proj_out, rows, dim, bits, st)); break;
    case 7: PHK_TRY(launch_ln_lfq<7>(x, gamma, beta, wp, bp, ids, out_norm, proj_out, rows, dim, bits, st)); break;
    default: PHK_TRY(launch_ln_lfq<8>(x, gamma, beta, wp, bp, ids, out_norm, proj_out, rows, dim, bits, st)); break;
  }
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_lfq_codes(const int64_t* ids, const float* w_out, const float* b_out, float* out, int64_t rows,
                             int32_t dim, int32_t bits, phk_stream_t s) {
  Prof prof_(FAM_LFQ, s, (double)rows * dim * 4.0);
  PHK_REQUIRE(ids && w_out && b_out && out, PHK_E_ARG, "phk_lfq_codes: null pointer");
  PHK_REQUIRE(rows >= 0 && dim > 0 && bits > 0 && bits <= 62, PHK_E_ARG, "phk_lfq_codes: bad size");
  if (rows == 0) return 0;
  const int64_t blocks = (rows * dim + 255) / 256;
  const unsigned grid = (unsigned)(blocks < (int64_t)kNumSMs * 16 ? blocks : kNumSMs * 16);
  PHK_CUDA(launch_pdl(lfq_codes_kernel, dim3(grid), dim3(256), (size_t)0, to_stream(s), ids, w_out, b_out, out, rows, dim, bits));
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_unpatchify(const float* P, int64_t ldp, float* video, int32_t B, int32_t C, int32_t F, int32_t H,
                              int32_t W, int32_t f0, int32_t nt, int32_t pt, int32_t p1, int32_t p2, phk_stream_t s) {
  Prof prof_(FAM_PATCHIFY, s, (double)B * C * nt * pt * H * W * 8.0);
  PHK_REQUIRE(P && video, PHK_E_ARG, "phk_unpatchify: null pointer");
  PHK_REQUIRE(B > 0 && C > 0 && F > 0 && H > 0 && W > 0 && pt > 0 && p1 > 0 && p2 > 0 && nt >= 0, PHK_E_ARG,
              "phk_unpatchify: bad size");
  PHK_REQUIRE(H % p1 == 0 && W % p2 == 0, PHK_E_SHAPE, "image size must be divisible by patch size (cvivit.py:271)");
  PHK_REQUIRE(f0 >= 0 && f0 + nt * pt <= F, PHK_E_SHAPE, "frame range outside the video");
  PHK_REQUIRE(ldp >= (int64_t)C * pt * p1 * p2, PHK_E_ARG, "phk_unpatchify: ldp smaller than the patch feature size");
  if (nt == 0) return 0;
  const bool vec = (p2 % 4 == 0) && (ldp % 4 == 0) && ((reinterpret_cast<uintptr_t>(video) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(P) & 15) == 0);
  const int64_t total = (int64_t)B * C * nt * pt * H * (W / (vec ? 4 : 1));
  const int64_t blocks = (total + 255) / 256;
  const unsigned grid = (unsigned)(blocks < (int64_t)kNumSMs * 16 ? blocks : kNumSMs * 16);
  if (vec) PHK_CUDA(launch_pdl(unpatchify_kernel<4>, dim3(grid), dim3(256), (size_t)0, to_stream(s), P, ldp, video, B, C, F, H, W, f0, nt, pt, p1, p2));
  else PHK_CUDA(launch_pdl(unpatchify_kernel<1>, dim3(grid), dim3(256), (size_t)0, to_stream(s), P, ldp, video, B, C, F, H, W, f0, nt, pt, p1, p2));
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_peg3d(const float* x, const float* w, const float* b, float* y, int32_t B, int32_t T, int32_t H,
                         int32_t W, int32_t D, int32_t causal, int32_t layout, phk_stream_t s) {
  Prof prof_(FAM_PEG, s, (double)B * T * H * W * D * 8.0);
  PHK_REQUIRE(x && w && b && y && x != y, PHK_E_ARG, "phk_peg3d: null or aliased pointer");
  PHK_REQUIRE(B > 0 && T > 0 && H > 0 && W > 0 && D > 0, PHK_E_ARG, "phk_peg3d: bad size");
  PHK_REQUIRE(D % 4 == 0, PHK_E_UNSUPPORTED, "phk_peg3d: dim must be a multiple of 4");
  const int64_t rows = (int64_t)B * T * H * W;
  PHK_REQUIRE(rows < (1LL << 31), PHK_E_UNSUPPORTED, "phk_peg3d: more than 2^31 positions");
  const int P = H * W;
  if (P <= 128 && D % PEG_CH == 0 && H <= 16 && (W == 4 || W == 8 || W == 16)) {
    const int pad = causal ? 2 : 1;
    if (W == 8) PHK_TRY(launch_peg_tiled<8>(x, w, b, y, B, T, H, D, pad, layout, to_stream(s)));
    else if (W == 4) PHK_TRY(launch_peg_tiled<4>(x, w, b, y, B, T, H, D, pad, layout, to_stream(s)));
    else PHK_TRY(launch_peg_tiled<16>(x, w, b, y, B, T, H, D, pad, layout, to_stream(s)));
  } else {
    PHK_CUDA(launch_pdl(peg_kernel, dim3((unsigned)rows), dim3(128), (size_t)(0), to_stream(s), x, w, b, y, T, H, W, D, causal ? 2 : 1, layout));
  }
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t phk_cpb_scratch_floats(const phk_cpb_t* c, int32_t d0, int32_t d1, int32_t d2) {
  if (!c || d0 <= 0 || d1 <= 0 || d2 <= 0) return 0;
  return (int64_t)(2 * d0 - 1) * (2 * d1 - 1) * (2 * d2 - 1) * c->heads;
}

extern "C" int phk_cpb_bias(const phk_cpb_t* c, int32_t d0, int32_t d1, int32_t d2, float* scratch, float* out,
                            phk_stream_t s) {
  Prof prof_(FAM_CPB, s);
  PHK_REQUIRE(c && scratch && out, PHK_E_ARG, "phk_cpb_bias: null pointer");
  PHK_REQUIRE(d0 > 0 && d1 > 0 && d2 > 0, PHK_E_ARG, "phk_cpb_bias: bad dims");
  PHK_REQUIRE(c->num_dims == 2 || c->num_dims == 3, PHK_E_UNSUPPORTED, "phk_cpb_bias: num_dims must be 2 or 3");
  PHK_REQUIRE(c->num_dims == 3 || d2 == 1, PHK_E_SHAPE, "phk_cpb_bias: 2-D bias needs d2 == 1");
  PHK_REQUIRE(c->hidden > 0 && c->hidden <= 4096 && c->heads > 0, PHK_E_UNSUPPORTED, "phk_cpb_bias: hidden > 4096");
  const int U = (2 * d0 - 1) * (2 * d1 - 1) * (2 * d2 - 1);
  PHK_CUDA(launch_pdl(cpb_table_kernel, dim3(U), dim3(256), (size_t)(2 * c->hidden * sizeof(float)), to_stream(s), *c, d0, d1, d2, scratch));
  PHK_LAUNCH_CHECK();
  const int64_t total = (int64_t)d0 * d1 * d2 * d0 * d1 * d2;
  const unsigned grid = (unsigned)((total + 255) / 256 < (int64_t)kNumSMs * 8 ? (total + 255) / 256 : kNumSMs * 8);
  PHK_CUDA(launch_pdl(cpb_expand_kernel, dim3(grid), dim3(256), (size_t)(0), to_stream(s), scratch, out, c->heads, d0, d1, d2));
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_sample_tokens(const float* cond, const float* null_logits, int64_t ld, const float* u,
                                 uint64_t seed, uint64_t offset, float cond_scale, float temperature,
                                 const uint8_t* mask, int64_t* ids, int64_t* pred_out, float* score_out, int64_t rows,
                                 int32_t V, int64_t seg_len, int64_t seg_stride, int64_t seg_off, phk_stream_t s) {
  Prof prof_(FAM_SAMPLE, s, (double)rows * V * 8.0);
  PHK_REQUIRE(cond, PHK_E_ARG, "phk_sample_tokens: null logits");
  PHK_REQUIRE(rows >= 0 && V > 0 && ld >= V, PHK_E_ARG, "phk_sample_tokens: bad size");
  if (rows == 0) return 0;
  const float* nul = (cond_scale == 1.0f) ? nullptr : null_logits;  // cond_scale == 1 returns logits (:157-158)
  PHK_REQUIRE(cond_scale == 1.0f || null_logits, PHK_E_ARG, "phk_sample_tokens: cond_scale != 1 needs null logits");
  const int threads = V >= 8192 ? 512 : (V >= 1024 ? 256 : 64);
  PHK_CUDA(launch_pdl(sample_tokens_kernel, dim3((unsigned)rows), dim3(threads), (size_t)(0), to_stream(s), cond, nul, ld, u, seed, offset, cond_scale, temperature, mask, ids, pred_out, score_out, V, seg_len, seg_stride, seg_off));
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_topk_mask(const float* scores, int32_t b, int32_t n, int32_t k, uint8_t* mask, int64_t* ids,
                             int64_t mask_id, phk_stream_t s) {
  Prof prof_(FAM_TOPK, s);
  PHK_REQUIRE(scores && mask && ids, PHK_E_ARG, "phk_topk_mask: null pointer");
  PHK_REQUIRE(b > 0 && n > 0 && n <= 8192, PHK_E_UNSUPPORTED, "phk_topk_mask: n must be in (0, 8192]");
  PHK_REQUIRE(k >= 0 && k <= n, PHK_E_SHAPE, "phk_topk_mask: k out of range (torch.topk would raise)");
  int threads = ((n + 31) / 32) * 32;
  if (threads > 1024) threads = 1024;
  PHK_CUDA(launch_pdl(topk_mask_kernel, dim3(b), dim3(threads), (size_t)(n * sizeof(float)), to_stream(s), scores, n, k, mask, ids, mask_id));
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_critic_scores(const float* x_cond, const float* x_null, const float* w, const float* b,
                                 const float* u, float cond_scale, float noise_K, float noise_mult, float* out,
                                 int64_t rows, int32_t dim, int64_t seg_len, int64_t seg_stride, int64_t seg_off,
                                 phk_stream_t s) {
  Prof prof_(FAM_CRITIC, s);
  PHK_REQUIRE(x_cond && w && b && out, PHK_E_ARG, "phk_critic_scores: null pointer");
  PHK_REQUIRE(rows >= 0 && dim > 0, PHK_E_ARG, "phk_critic_scores: bad size");
  if (rows == 0) return 0;
  const float* xn = (cond_scale == 1.0f) ? nullptr : x_null;
  PHK_REQUIRE(cond_scale == 1.0f || x_null, PHK_E_ARG, "phk_critic_scores: cond_scale != 1 needs the null pass");
  PHK_CUDA(launch_pdl(critic_scores_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), (size_t)(0), to_stream(s), x_cond, xn, w, b, u, cond_scale, noise_K, noise_mult, out, rows, dim, seg_len, seg_stride, seg_off));
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int phk_cfg_combine(const float* cond, const float* null_out, float cond_scale, float* out, int64_t n,
                               phk_stream_t s) {
  Prof prof_(FAM_CFG, s);
  PHK_REQUIRE(cond && null_out && out, PHK_E_ARG, "phk_cfg_combine: null pointer");
  PHK_REQUIRE(n >= 0, PHK_E_ARG, "phk_cfg_combine: bad size");
  if (n == 0) return 0;
  const int64_t blocks = (n + 255) / 256;
  PHK_CUDA(launch_pdl(cfg_combine_kernel, dim3((unsigned)(blocks < (int64_t)kNumSMs * 16 ? blocks : kNumSMs * 16)), dim3(256), (size_t)(0), to_stream(s), cond, null_out, cond_scale, out, n));
  PHK_LAUNCH_CHECK();
  return 0;
}
