// Cosine-sim multi-head attention core, fp32 (attention.py:146-181), all four uses of the
// reference with one kernel: C-ViViT spatial (bias), C-ViViT temporal (causal + ALiBi),
// MaskGit self (3-D bias, optional key mask), cross (null-kv, text mask, CFG half dropped).
//
// Flash-style: one CTA per (query tile of 64, head, sequence); keys/values streamed in
// chunks of 64 through shared memory with an online softmax, S and P never touch HBM.
//   q,k  : l2-normalised over dim_head (F.normalize, eps 1e-12) then * q_scale / k_scale
//   sim  : q.k * scale (+ bias) ; key mask / causal -> -FLT_MAX ; softmax ; . v
// Sequences are addressed with (outer, inner, token) strides so neither the spatial
// '(b t)(h w)' nor the temporal '(b h w) t' view is ever materialised (cvivit.py:458,468).
#include "phk_common.cuh"

namespace phk {

constexpr int TQ = 64, TK = 64, ATT_THREADS = 256;

template <int DH>
struct AttSmem {
  float q[DH][TQ + 4];   // d-major (transposed) normalised queries
  float k[DH][TK + 4];   // d-major normalised keys of the current chunk
  float v[TK][DH + 4];   // values of the current chunk
  float p[TQ][TK + 4];   // probabilities of the current chunk
};

template <int DH>
__global__ void __launch_bounds__(ATT_THREADS) attention_kernel(const float* __restrict__ q,
                                                                const float* __restrict__ kv,
                                                                const float* __restrict__ null_kv,
                                                                const float* __restrict__ q_scale,
                                                                const float* __restrict__ k_scale,
                                                                const float* __restrict__ bias,
                                                                const uint8_t* __restrict__ key_mask,
                                                                const float* __restrict__ alibi_slopes,
                                                                void* __restrict__ out, phk_attn_geom_t g) {
  pdl_prologue();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  AttSmem<DH>& sm = *reinterpret_cast<AttSmem<DH>*>(smem_raw);
  const int qt = blockIdx.x, h = blockIdx.y, seq = blockIdx.z;
  const int so = seq / g.n_inner, si = seq - so * g.n_inner;
  const int kv_so = g.kv_outer_mod > 0 ? so % g.kv_outer_mod : so;
  const int mask_row = g.mask_outer_mod > 0 ? so % g.mask_outer_mod : so;
  const bool mask_dropped = g.mask_off_from >= 0 && so >= g.mask_off_from;
  const int I = g.heads * DH;
  const int nnull = g.num_null_kv;
  const int nk_total = g.n_k + nnull;
  const int q0 = qt * TQ;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;

  const float* qbase = q + (int64_t)so * g.q_outer + (int64_t)si * g.q_inner + (int64_t)h * DH;
  const float* kbase = kv + (int64_t)kv_so * g.k_outer + (int64_t)si * g.k_inner + (int64_t)h * DH;

  // ---- load + normalise the query tile (warp per row, lanes over d) ----
  constexpr int DPL = (DH + 31) / 32;  // d's per lane
  for (int r = wid; r < TQ; r += ATT_THREADS / 32) {
    const int qi = q0 + r;
    float x[DPL];
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < DPL; ++c) {
      const int d = lane + 32 * c;
      x[c] = (qi < g.n_q && d < DH) ? qbase[(int64_t)qi * g.q_tok + d] : 0.f;
      ss += x[c] * x[c];
    }
    const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
    for (int c = 0; c < DPL; ++c) {
      const int d = lane + 32 * c;
      if (d < DH) sm.q[d][r] = (x[c] / nrm) * q_scale[d];
    }
  }

  float m_run[4], l_run[4];
  constexpr int CW = DH / 16;  // output columns per thread
  float o_acc[4][CW];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_run[i] = -INFINITY;
    l_run[i] = 0.f;
#pragma unroll
    for (int c = 0; c < CW; ++c) o_acc[i][c] = 0.f;
  }
  const float slope = (g.causal && alibi_slopes) ? alibi_slopes[h] : 0.f;
  const int row_shift = g.n_k - g.n_q;  // query i sits at key position i + (j - i) (attention.py:196)

  for (int j0 = 0; j0 < nk_total; j0 += TK) {
    __syncthreads();  // previous chunk fully consumed (also orders the q tile on the first pass)
    // ---- load key / value chunk ----
    for (int r = wid; r < TK; r += ATT_THREADS / 32) {
      const int jj = j0 + r;
      const float* kp = nullptr;
      const float* vp = nullptr;
      if (jj < nnull) {
        kp = null_kv + ((int64_t)h * 2 * nnull + 2 * jj) * DH;  // 'h (n r) d', r=0 key, r=1 value (:148)
        vp = kp + DH;
      } else if (jj < nk_total) {
        kp = kbase + (int64_t)(jj - nnull) * g.k_tok;
        vp = kp + I;
      }
      float x[DPL];
      float ss = 0.f;
#pragma unroll
      for (int c = 0; c < DPL; ++c) {
        const int d = lane + 32 * c;
        x[c] = (kp && d < DH) ? kp[d] : 0.f;
        ss += x[c] * x[c];
        if (d < DH) sm.v[r][d] = vp ? vp[d] : 0.f;
      }
      const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
      for (int c = 0; c < DPL; ++c) {
        const int d = lane + 32 * c;
        if (d < DH) sm.k[d][r] = (x[c] / nrm) * k_scale[d];
      }
    }
    __syncthreads();
    // ---- S = q k^T ----
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
    for (int d = 0; d < DH; ++d) {
      const float4 a = *reinterpret_cast<const float4*>(&sm.q[d][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&sm.k[d][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(av[i], bv[j], s[i][j]);
    }
    // ---- scale, bias, masks, online softmax ----
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int qi = q0 + ty * 4 + i;
      float rmax = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int jj = j0 + tx * 4 + j;
        float val = s[i][j] * g.scale;
        if (jj >= nk_total || qi >= g.n_q) {
          val = -INFINITY;  // padding, contributes nothing
        } else {
          const int kj = jj - nnull;  // index among the real keys
          if (bias && kj >= 0) val += bias[((int64_t)h * g.n_q + qi) * g.n_k + kj];
          if (key_mask && kj >= 0 && (mask_dropped || !key_mask[(int64_t)mask_row * g.n_k + kj])) val = -FLT_MAX;
          if (g.causal) {
            const int pos = qi + row_shift;
            val += -fabsf((float)(jj - pos)) * slope;
            if (jj > pos) val = -FLT_MAX;
          }
        }
        s[i][j] = val;
        rmax = fmaxf(rmax, val);
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) rmax = fmaxf(rmax, __shfl_xor_sync(0xffffffffu, rmax, o));
      const float m_new = fmaxf(m_run[i], rmax);
      const float m_use = (m_new == -INFINITY) ? 0.f : m_new;  // fully padded query row
      const float corr = expf(m_run[i] - m_use);
      float rsum = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float pv = expf(s[i][j] - m_use);
        rsum += pv;
        sm.p[ty * 4 + i][tx * 4 + j] = pv;
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) rsum += __shfl_xor_sync(0xffffffffu, rsum, o);
      l_run[i] = l_run[i] * corr + rsum;
      m_run[i] = m_new;
#pragma unroll
      for (int c = 0; c < CW; ++c) o_acc[i][c] *= corr;
    }
    __syncthreads();
    // ---- O += P V ----
#pragma unroll 4
    for (int j = 0; j < TK; ++j) {
      float vv[CW];
#pragma unroll
      for (int c = 0; c < CW; ++c) vv[c] = sm.v[j][tx * CW + c];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float pv = sm.p[ty * 4 + i][j];
#pragma unroll
        for (int c = 0; c < CW; ++c) o_acc[i][c] = fmaf(pv, vv[c], o_acc[i][c]);
      }
    }
  }
  // ---- normalise and store 'b h n d -> b n (h d)' (:181) ----
  const int64_t obase = (int64_t)so * g.o_outer + (int64_t)si * g.o_inner + (int64_t)h * DH;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int qi = q0 + ty * 4 + i;
    if (qi >= g.n_q) continue;
    const float inv = 1.f / l_run[i];
#pragma unroll
    for (int c = 0; c < CW; ++c) {
      const float ov = o_acc[i][c] * inv;
      const int64_t off = obase + (int64_t)qi * g.o_tok + tx * CW + c;
      if (g.out_bf16) reinterpret_cast<__nv_bfloat16*>(out)[off] = __float2bfloat16_rn(ov);
      else reinterpret_cast<float*>(out)[off] = ov;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Short sequences (n <= 16): the C-ViViT temporal transformer attends over T' = 9 tokens
// (cvivit.py:468-470), 4096 (sequence, head) pairs per layer at config 2.  A 64-wide tile would be
// 98 % padding, so here ONE WARP owns one (sequence, head): q/k/v rows live in registers (lane = d),
// normalised q/k are staged in 2 x n x (DH+1) floats of shared memory for the n*n dot products,
// softmax runs one row per lane, and P.V accumulates back in registers.  No tensor tile on purpose.
// ------------------------------------------------------------------------------------------
constexpr int SMALL_N = 16, SMALL_WARPS = 8;

// NMAX: compile-time bound of the unrolled row loops (the exact n of the workload when possible: no predicated-off slots)
template <int DH, int NMAX>
__global__ void __launch_bounds__(SMALL_WARPS * 32) attention_small_kernel(
    const float* __restrict__ q, const float* __restrict__ kv, const float* __restrict__ q_scale,
    const float* __restrict__ k_scale, const float* __restrict__ alibi_slopes, void* __restrict__ out,
    phk_attn_geom_t g) {
  pdl_prologue();
  constexpr int DPL = DH / 32;
  constexpr int LDQ = DH + 1;
  extern __shared__ float small_smem[];  // per warp: q[n][DH+1], k[n][DH+1], p[n][n+1] (sized by the actual n)
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int LDP = g.n_q + 1;
  float* s_q = small_smem + (size_t)w * (2 * g.n_q * LDQ + g.n_q * LDP);
  float* s_k = s_q + g.n_q * LDQ;
  float* s_p = s_k + g.n_q * LDQ;
  const int64_t pair = (int64_t)blockIdx.x * SMALL_WARPS + w;
  const int64_t npairs = (int64_t)g.n_outer * g.n_inner * g.heads;
  if (pair >= npairs) return;  // whole warp exits together
  const int h = (int)(pair % g.heads);
  const int seq = (int)(pair / g.heads);
  const int so = seq / g.n_inner, si = seq - so * g.n_inner;
  const int n = g.n_q, I = g.heads * DH;
  const float* qb = q + (int64_t)so * g.q_outer + (int64_t)si * g.q_inner + (int64_t)h * DH;
  const float* kb = kv + (int64_t)so * g.k_outer + (int64_t)si * g.k_inner + (int64_t)h * DH;
  float qs[DPL], ks[DPL];
#pragma unroll
  for (int c = 0; c < DPL; ++c) { qs[c] = q_scale[lane + 32 * c]; ks[c] = k_scale[lane + 32 * c]; }
  float v[NMAX][DPL], xq[NMAX][DPL], xk[NMAX][DPL];
  // all 3n row loads are issued before the first reduction (one exposed memory latency instead of n)
#pragma unroll
  for (int i = 0; i < NMAX; ++i) {
#pragma unroll
    for (int c = 0; c < DPL; ++c) {
      const bool in = i < n;
      xq[i][c] = in ? qb[(int64_t)i * g.q_tok + lane + 32 * c] : 0.f;
      xk[i][c] = in ? kb[(int64_t)i * g.k_tok + lane + 32 * c] : 0.f;
      v[i][c] = in ? kb[(int64_t)i * g.k_tok + I + lane + 32 * c] : 0.f;
    }
  }
#pragma unroll
  for (int i = 0; i < NMAX; ++i) {
    if (i < n) {
      float sq = 0.f, sk = 0.f;
#pragma unroll
      for (int c = 0; c < DPL; ++c) { sq += xq[i][c] * xq[i][c]; sk += xk[i][c] * xk[i][c]; }
      const float nq = fmaxf(sqrtf(warp_sum(sq)), 1e-12f), nk = fmaxf(sqrtf(warp_sum(sk)), 1e-12f);
#pragma unroll
      for (int c = 0; c < DPL; ++c) {
        s_q[i * LDQ + lane + 32 * c] = (xq[i][c] / nq) * qs[c];
        s_k[i * LDQ + lane + 32 * c] = (xk[i][c] / nk) * ks[c];
      }
    }
  }
  __syncwarp();
  // scores: lanes stride over the n*n (i, j) pairs
  const float slope = (g.causal && alibi_slopes) ? alibi_slopes[h] : 0.f;
  for (int p = lane; p < n * n; p += 32) {
    const int i = p / n, j = p - i * n;
    float acc = 0.f;
    if (!g.causal || j <= i) {
#pragma unroll 16
      for (int d = 0; d < DH; ++d) acc = fmaf(s_q[i * LDQ + d], s_k[j * LDQ + d], acc);
      acc *= g.scale;
      if (g.causal) acc += -fabsf((float)(j - i)) * slope;
    } else {
      acc = -FLT_MAX;
    }
    s_p[i * LDP + j] = acc;
  }
  __syncwarp();
  if (lane < n) {  // softmax, one row per lane
    float m = -FLT_MAX;
    for (int j = 0; j < n; ++j) m = fmaxf(m, s_p[lane * LDP + j]);
    float sum = 0.f;
    for (int j = 0; j < n; ++j) { const float e = expf(s_p[lane * LDP + j] - m); s_p[lane * LDP + j] = e; sum += e; }
    const float inv = 1.f / sum;
    for (int j = 0; j < n; ++j) s_p[lane * LDP + j] *= inv;
  }
  __syncwarp();
  const int64_t ob = (int64_t)so * g.o_outer + (int64_t)si * g.o_inner + (int64_t)h * DH;
#pragma unroll
  for (int i = 0; i < NMAX; ++i) {
    if (i < n) {
      float o[DPL];
#pragma unroll
      for (int c = 0; c < DPL; ++c) o[c] = 0.f;
#pragma unroll
      for (int j = 0; j < NMAX; ++j) {
        if (j < n) {
          const float pv = s_p[i * LDP + j];
#pragma unroll
          for (int c = 0; c < DPL; ++c) o[c] = fmaf(pv, v[j][c], o[c]);
        }
      }
#pragma unroll
      for (int c = 0; c < DPL; ++c) {
        const int64_t off = ob + (int64_t)i * g.o_tok + lane + 32 * c;
        if (g.out_bf16) reinterpret_cast<__nv_bfloat16*>(out)[off] = __float2bfloat16_rn(o[c]);
        else reinterpret_cast<float*>(out)[off] = o[c];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Few keys (null-kv + text length <= 64): MaskGit / TokenCritic cross-attention over the T5 context
// (attention.py:137-168 with num_null_kv = 2).  A 64-wide key tile would be ~70 % padding, so the mapping is turned
// around: ONE THREAD OWNS ONE QUERY.  Its normalised query (dim_head registers) meets every key / value as a
// shared-memory BROADCAST (all lanes read the same address), i.e. ~2.5 issue slots per (query, key) dot product
// instead of ~10 with a lane=d or lane=key mapping.  Two passes over the (few) keys: scores + row max (scores parked
// in shared memory), then p = exp(s - m), sum and P.V -- no online rescale of the dim_head-wide accumulator.
// ------------------------------------------------------------------------------------------
// 4 threads split dim_head, and every thread carries QPT queries so that each 16-byte key / value chunk read from
// shared memory feeds QPT x 4 FMAs (the kernel is shared-memory-bandwidth bound otherwise: LDS.128 = 4 wavefronts)
constexpr int FEW_KEYS = 64, FEW_THREADS = 128, TPQ = 4, QPT = 4;
constexpr int FEW_QUERIES = FEW_THREADS / TPQ * QPT;  // 128 queries per CTA

template <int DH>
__global__ void __launch_bounds__(FEW_THREADS) attention_fewkeys_kernel(
    const float* __restrict__ q, const float* __restrict__ kv, const float* __restrict__ null_kv,
    const float* __restrict__ q_scale, const float* __restrict__ k_scale, const uint8_t* __restrict__ key_mask,
    void* __restrict__ out, phk_attn_geom_t g) {
  pdl_prologue();
  constexpr int DPL = DH / 32;
  constexpr int DP = DH / TPQ;  // d's per thread
  extern __shared__ __align__(16) float few_smem[];
  const int I = g.heads * DH, nnull = g.num_null_kv, nk_all = g.n_k + nnull;
  float* s_k = few_smem;                  // [nk][DH]
  float* s_v = s_k + nk_all * DH;             // [nk][DH]
  float* s_s = s_v + nk_all * DH;             // [nk][FEW_QUERIES] scores, one column per query
  float* s_flag = s_s + nk_all * FEW_QUERIES; // [nk] 0: live key, -FLT_MAX: masked (masked_fill(~mask, -finfo.max), :168)
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int h = blockIdx.y, seq = blockIdx.z;
  const int so = seq / g.n_inner, si = seq - so * g.n_inner;
  const int kv_so = g.kv_outer_mod > 0 ? so % g.kv_outer_mod : so;
  const int mask_row = g.mask_outer_mod > 0 ? so % g.mask_outer_mod : so;
  const bool mask_dropped = g.mask_off_from >= 0 && so >= g.mask_off_from;
  // The null half of a classifier-free-guidance pair sees no text at all (every context key masked,
  // phenaki_pytorch.py:188-190): only the null keys are live.  A masked key contributes exp(-FLT_MAX - m) = 0 exactly,
  // so leaving the dead keys out gives the same bits with 1/9 of the work (2 of 18 keys at L = 16).
  const int nk = (mask_dropped && key_mask && nnull > 0) ? nnull : nk_all;
  const float* kbase = kv + (int64_t)kv_so * g.k_outer + (int64_t)si * g.k_inner + (int64_t)h * DH;
  for (int j = w; j < nk; j += FEW_THREADS / 32) {  // warp per key: l2-normalise, * k_scale
    const float* kp;
    const float* vp;
    if (j < nnull) { kp = null_kv + ((int64_t)h * 2 * nnull + 2 * j) * DH; vp = kp + DH; }   // 'h (n r) d' (:148)
    else { kp = kbase + (int64_t)(j - nnull) * g.k_tok; vp = kp + I; }
    float x[DPL], ss = 0.f;
#pragma unroll
    for (int c = 0; c < DPL; ++c) { x[c] = kp[lane + 32 * c]; ss += x[c] * x[c]; s_v[j * DH + lane + 32 * c] = vp[lane + 32 * c]; }
    const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
    for (int c = 0; c < DPL; ++c) s_k[j * DH + lane + 32 * c] = (x[c] / nrm) * k_scale[lane + 32 * c];
    if (lane == 0) {
      const int kj = j - nnull;
      const bool dead = key_mask && kj >= 0 && (mask_dropped || !key_mask[(int64_t)mask_row * g.n_k + kj]);
      s_flag[j] = dead ? -FLT_MAX : 0.f;
    }
  }
  __syncthreads();
  const int tg = threadIdx.x / TPQ, part = threadIdx.x % TPQ;
  const int ql0 = tg * QPT;                               // first local query of this thread group
  const int q0 = blockIdx.x * FEW_QUERIES + ql0;
  float qv[QPT][DP];
  float ss[QPT];
  const float* qbase = q + (int64_t)so * g.q_outer + (int64_t)si * g.q_inner + (int64_t)h * DH + part * DP;
#pragma unroll
  for (int u = 0; u < QPT; ++u) {
    ss[u] = 0.f;
    const bool valid = q0 + u < g.n_q;
#pragma unroll
    for (int c = 0; c < DP / 4; ++c) {
      const float4 t = valid ? reinterpret_cast<const float4*>(qbase + (int64_t)(q0 + u) * g.q_tok)[c] : make_float4(0.f, 0.f, 0.f, 0.f);
      qv[u][4 * c] = t.x; qv[u][4 * c + 1] = t.y; qv[u][4 * c + 2] = t.z; qv[u][4 * c + 3] = t.w;
      ss[u] += (t.x * t.x + t.y * t.y) + (t.z * t.z + t.w * t.w);
    }
  }
#pragma unroll
  for (int u = 0; u < QPT; ++u) {
    ss[u] += __shfl_xor_sync(0xffffffffu, ss[u], 1);
    ss[u] += __shfl_xor_sync(0xffffffffu, ss[u], 2);
    const float inv_n = g.scale / fmaxf(sqrtf(ss[u]), 1e-12f);
#pragma unroll
    for (int d = 0; d < DP; ++d) qv[u][d] = qv[u][d] * inv_n * q_scale[part * DP + d];
  }
  // pass 1: scores and row maxima; every key chunk read from shared memory is used by QPT queries
  float m[QPT];
#pragma unroll
  for (int u = 0; u < QPT; ++u) m[u] = -INFINITY;
  for (int j = 0; j < nk; ++j) {
    const float4* kr = reinterpret_cast<const float4*>(s_k + j * DH + part * DP);
    float a[QPT];
#pragma unroll
    for (int u = 0; u < QPT; ++u) a[u] = 0.f;
#pragma unroll
    for (int c = 0; c < DP / 4; ++c) {
      const float4 kk = kr[c];
#pragma unroll
      for (int u = 0; u < QPT; ++u) {
        a[u] = fmaf(qv[u][4 * c], kk.x, a[u]); a[u] = fmaf(qv[u][4 * c + 1], kk.y, a[u]);
        a[u] = fmaf(qv[u][4 * c + 2], kk.z, a[u]); a[u] = fmaf(qv[u][4 * c + 3], kk.w, a[u]);
      }
    }
    const bool dead = s_flag[j] != 0.f;
#pragma unroll
    for (int u = 0; u < QPT; ++u) {
      float sc = a[u];
      sc += __shfl_xor_sync(0xffffffffu, sc, 1);
      sc += __shfl_xor_sync(0xffffffffu, sc, 2);
      if (dead) sc = -FLT_MAX;
      if (part == u) s_s[j * FEW_QUERIES + ql0 + u] = sc;  // spread the QPT stores over the 4 threads of the group
      m[u] = fmaxf(m[u], sc);
    }
  }
  __syncwarp();
  // pass 2: p = exp(s - m), l = sum p, o = sum p * v  (the query registers are reused as the output accumulators)
  float l[QPT];
#pragma unroll
  for (int u = 0; u < QPT; ++u) {
    l[u] = 0.f;
#pragma unroll
    for (int d = 0; d < DP; ++d) qv[u][d] = 0.f;
  }
  for (int j = 0; j < nk; ++j) {
    const float4 s4 = *reinterpret_cast<const float4*>(s_s + j * FEW_QUERIES + ql0);
    const float pj[QPT] = {__expf(s4.x - m[0]), __expf(s4.y - m[1]), __expf(s4.z - m[2]), __expf(s4.w - m[3])};
    const float4* vr = reinterpret_cast<const float4*>(s_v + j * DH + part * DP);
#pragma unroll
    for (int u = 0; u < QPT; ++u) l[u] += pj[u];
#pragma unroll
    for (int c = 0; c < DP / 4; ++c) {
      const float4 vv = vr[c];
#pragma unroll
      for (int u = 0; u < QPT; ++u) {
        qv[u][4 * c] = fmaf(pj[u], vv.x, qv[u][4 * c]); qv[u][4 * c + 1] = fmaf(pj[u], vv.y, qv[u][4 * c + 1]);
        qv[u][4 * c + 2] = fmaf(pj[u], vv.z, qv[u][4 * c + 2]); qv[u][4 * c + 3] = fmaf(pj[u], vv.w, qv[u][4 * c + 3]);
      }
    }
  }
#pragma unroll
  for (int u = 0; u < QPT; ++u) {
    if (q0 + u >= g.n_q) continue;
    const float inv = 1.f / l[u];
    const int64_t off = (int64_t)so * g.o_outer + (int64_t)si * g.o_inner + (int64_t)(q0 + u) * g.o_tok + (int64_t)h * DH + part * DP;
    if (g.out_bf16) {
      __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(out) + off;
#pragma unroll
      for (int c = 0; c < DP / 8; ++c)
        reinterpret_cast<uint4*>(op)[c] = make_uint4(pack_bf16x2(qv[u][8 * c] * inv, qv[u][8 * c + 1] * inv),
                                                      pack_bf16x2(qv[u][8 * c + 2] * inv, qv[u][8 * c + 3] * inv),
                                                      pack_bf16x2(qv[u][8 * c + 4] * inv, qv[u][8 * c + 5] * inv),
                                                      pack_bf16x2(qv[u][8 * c + 6] * inv, qv[u][8 * c + 7] * inv));
    } else {
      float* op = reinterpret_cast<float*>(out) + off;
#pragma unroll
      for (int c = 0; c < DP / 4; ++c)
        reinterpret_cast<float4*>(op)[c] = make_float4(qv[u][4 * c] * inv, qv[u][4 * c + 1] * inv, qv[u][4 * c + 2] * inv, qv[u][4 * c + 3] * inv);
    }
  }
}

template <int DH>
static int launch_attention_fewkeys(const float* q, const float* kv, const float* null_kv, const float* q_scale,
                                    const float* k_scale, const uint8_t* key_mask, void* out, const phk_attn_geom_t& g,
                                    cudaStream_t st) {
  const int nk = g.n_k + g.num_null_kv;
  const size_t smem = (size_t)(2 * nk * DH + nk * FEW_QUERIES + nk) * sizeof(float);
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(attention_fewkeys_kernel<DH>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)((2 * FEW_KEYS * DH + FEW_KEYS * FEW_QUERIES + FEW_KEYS) * sizeof(float))));
    mark_configured(&configured_mask);
  }
  dim3 grid((unsigned)((g.n_q + FEW_QUERIES - 1) / FEW_QUERIES), (unsigned)g.heads, (unsigned)(g.n_outer * g.n_inner));
  PHK_CUDA(launch_pdl(attention_fewkeys_kernel<DH>, grid, dim3(FEW_THREADS), smem, st, q, kv, null_kv, q_scale, k_scale,
                      key_mask, out, g));
  PHK_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------
// Short sequences, thread-per-query variant (the one used): a CTA holds G = 128 / n (sequence, head) groups; thread
// (group, i) owns query i AND stages key / value row i of its group (each thread normalises its own rows: no
// shuffles).  Scores, softmax and P.V then run entirely in registers against the group's keys / values in shared
// memory -- ~1500 issue slots per 32 queries instead of per 9.
// ------------------------------------------------------------------------------------------
constexpr int ROWS_THREADS = 256, ROWS_QUERIES = ROWS_THREADS / 4;
template <int DH, int NMAX>
__global__ void __launch_bounds__(ROWS_THREADS) attention_rows_kernel(const float* __restrict__ q, const float* __restrict__ kv,
                                                                      const float* __restrict__ q_scale,
                                                                      const float* __restrict__ k_scale,
                                                                      const float* __restrict__ alibi_slopes,
                                                                      void* __restrict__ out, phk_attn_geom_t g) {
  pdl_prologue();
  constexpr int DP = DH / 4;  // 4 threads share one query / one staged key+value row
  extern __shared__ __align__(16) float rows_smem[];  // [G][n*DH + 16] keys, then the same for values
  const int n = g.n_q, G = ROWS_QUERIES / n;
  const int GS = n * DH + 16;  // group stride: the +16 floats stagger the banks of neighbouring groups
  const int ql = threadIdx.x >> 2, part = threadIdx.x & 3;
  const int grp = ql / n, i = ql - grp * n;
  const int64_t pair = (int64_t)blockIdx.x * G + grp;
  const int64_t npairs = (int64_t)g.n_outer * g.n_inner * g.heads;
  const bool active = grp < G && pair < npairs;
  float* s_k = rows_smem + (size_t)(grp < G ? grp : 0) * GS;
  float* s_v = rows_smem + (size_t)G * GS + (size_t)(grp < G ? grp : 0) * GS;
  const int I = g.heads * DH;
  float qv[DP];
  float4 kr[DP / 4];
  int h = 0;
  int64_t obase = 0;
  float sq = 0.f, sk = 0.f;
  if (active) {
    h = (int)(pair % g.heads);
    const int seq = (int)(pair / g.heads);
    const int so = seq / g.n_inner, si = seq - so * g.n_inner;
    const float4* qp = reinterpret_cast<const float4*>(q + (int64_t)so * g.q_outer + (int64_t)si * g.q_inner +
                                                       (int64_t)i * g.q_tok + (int64_t)h * DH + part * DP);
    const float4* kp = reinterpret_cast<const float4*>(kv + (int64_t)so * g.k_outer + (int64_t)si * g.k_inner +
                                                       (int64_t)i * g.k_tok + (int64_t)h * DH + part * DP);
    const float4* vp = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(kp) + I);
    obase = (int64_t)so * g.o_outer + (int64_t)si * g.o_inner + (int64_t)i * g.o_tok + (int64_t)h * DH + part * DP;
#pragma unroll
    for (int c = 0; c < DP / 4; ++c) {
      const float4 t = qp[c];
      qv[4 * c] = t.x; qv[4 * c + 1] = t.y; qv[4 * c + 2] = t.z; qv[4 * c + 3] = t.w;
      sq += (t.x * t.x + t.y * t.y) + (t.z * t.z + t.w * t.w);
      kr[c] = kp[c];
      sk += (kr[c].x * kr[c].x + kr[c].y * kr[c].y) + (kr[c].z * kr[c].z + kr[c].w * kr[c].w);
      reinterpret_cast<float4*>(s_v + i * DH + part * DP)[c] = vp[c];
    }
  } else {
#pragma unroll
    for (int d = 0; d < DP; ++d) qv[d] = 0.f;
#pragma unroll
    for (int c = 0; c < DP / 4; ++c) kr[c] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  sq += __shfl_xor_sync(0xffffffffu, sq, 1); sq += __shfl_xor_sync(0xffffffffu, sq, 2);
  sk += __shfl_xor_sync(0xffffffffu, sk, 1); sk += __shfl_xor_sync(0xffffffffu, sk, 2);
  if (active) {
    const float iq = g.scale / fmaxf(sqrtf(sq), 1e-12f), ik = 1.f / fmaxf(sqrtf(sk), 1e-12f);
#pragma unroll
    for (int c = 0; c < DP / 4; ++c) {
      const float4 ks = *reinterpret_cast<const float4*>(k_scale + part * DP + 4 * c);
      reinterpret_cast<float4*>(s_k + i * DH + part * DP)[c] =
          make_float4(kr[c].x * ik * ks.x, kr[c].y * ik * ks.y, kr[c].z * ik * ks.z, kr[c].w * ik * ks.w);
      const float4 qs = *reinterpret_cast<const float4*>(q_scale + part * DP + 4 * c);
      qv[4 * c] *= iq * qs.x; qv[4 * c + 1] *= iq * qs.y; qv[4 * c + 2] *= iq * qs.z; qv[4 * c + 3] *= iq * qs.w;
    }
  }
  __syncthreads();
  const float slope = (g.causal && alibi_slopes && active) ? alibi_slopes[h] : 0.f;
  float sc[NMAX];
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < NMAX; ++j) {
    float a0 = 0.f, a1 = 0.f;
    if (j < n) {
      const float4* krow = reinterpret_cast<const float4*>(s_k + j * DH + part * DP);
#pragma unroll
      for (int c = 0; c < DP / 4; ++c) {
        const float4 kk = krow[c];
        a0 = fmaf(qv[4 * c], kk.x, a0); a1 = fmaf(qv[4 * c + 1], kk.y, a1);
        a0 = fmaf(qv[4 * c + 2], kk.z, a0); a1 = fmaf(qv[4 * c + 3], kk.w, a1);
      }
    }
    float sj = a0 + a1;
    sj += __shfl_xor_sync(0xffffffffu, sj, 1);
    sj += __shfl_xor_sync(0xffffffffu, sj, 2);
    const bool live = j < n && (!g.causal || j <= i);
    if (g.causal) sj += -fabsf((float)(j - i)) * slope;  // ALiBi (attention.py:170-174)
    sc[j] = live ? sj : -INFINITY;
    m = fmaxf(m, sc[j]);
  }
  if (!active) return;
  float l = 0.f;
#pragma unroll
  for (int d = 0; d < DP; ++d) qv[d] = 0.f;  // reuse as the output accumulator
#pragma unroll
  for (int j = 0; j < NMAX; ++j) {
    if (j < n && (!g.causal || j <= i)) {
      const float pj = __expf(sc[j] - m);
      l += pj;
      const float4* vr = reinterpret_cast<const float4*>(s_v + j * DH + part * DP);
#pragma unroll
      for (int c = 0; c < DP / 4; ++c) {
        const float4 vv = vr[c];
        qv[4 * c] = fmaf(pj, vv.x, qv[4 * c]); qv[4 * c + 1] = fmaf(pj, vv.y, qv[4 * c + 1]);
        qv[4 * c + 2] = fmaf(pj, vv.z, qv[4 * c + 2]); qv[4 * c + 3] = fmaf(pj, vv.w, qv[4 * c + 3]);
      }
    }
  }
  const float inv = 1.f / l;
  if (g.out_bf16) {
    __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(out) + obase;
#pragma unroll
    for (int c = 0; c < DP / 8; ++c)
      reinterpret_cast<uint4*>(op)[c] = make_uint4(pack_bf16x2(qv[8 * c] * inv, qv[8 * c + 1] * inv),
                                                    pack_bf16x2(qv[8 * c + 2] * inv, qv[8 * c + 3] * inv),
                                                    pack_bf16x2(qv[8 * c + 4] * inv, qv[8 * c + 5] * inv),
                                                    pack_bf16x2(qv[8 * c + 6] * inv, qv[8 * c + 7] * inv));
  } else {
    float* op = reinterpret_cast<float*>(out) + obase;
#pragma unroll
    for (int c = 0; c < DP / 4; ++c)
      reinterpret_cast<float4*>(op)[c] = make_float4(qv[4 * c] * inv, qv[4 * c + 1] * inv, qv[4 * c + 2] * inv, qv[4 * c + 3] * inv);
  }
}

// ------------------------------------------------------------------------------------------
// Short self-attention sequences with dim_head 64 (temporal axis of C-ViViT: n = T' = 9, causal + ALiBi,
// attention.py:128-182, 186-227): one WARP per (sequence, head), nothing staged in shared memory.  Lane l holds dims
// (2l, 2l+1) of every token's q, k and v (3n coalesced 256-B row loads, all in flight together); cosine-sim
// normalisation, the n(n+1)/2 causal dot products and the softmax run on warp shuffles, the P.V product is two FMAs
// per (i, j) and lane.  33 MB of q / kv / out traffic at cfg2 bound the kernel, not shuffles (~0.3 k per warp).
// ------------------------------------------------------------------------------------------
// PRE: q / kv are the bf16 operands phk_gemm_bf16_qkv writes (already l2-normalised, scaled, similarity scale folded
// into q): half the bytes to read and no normalisation shuffles.
template <int NMAX, bool PRE = false>
__global__ void __launch_bounds__(256) attention_warp64_kernel(const void* __restrict__ q_, const void* __restrict__ kv_,
                                                               const float* __restrict__ q_scale,
                                                               const float* __restrict__ k_scale,
                                                               const float* __restrict__ alibi_slopes,
                                                               void* __restrict__ out, phk_attn_geom_t g) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t pair = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t npairs = (int64_t)g.n_outer * g.n_inner * g.heads;
  if (pair >= npairs) return;  // whole warp exits together
  const int h = (int)(pair % g.heads);
  const int seq = (int)(pair / g.heads);
  const int so = seq / g.n_inner, si = seq - so * g.n_inner;
  const int n = g.n_q, I = g.heads * 64;
  float2 xq[NMAX], xk[NMAX], xv[NMAX];
  const int64_t qoff = (int64_t)so * g.q_outer + (int64_t)si * g.q_inner + (int64_t)h * 64;
  const int64_t koff = (int64_t)so * g.k_outer + (int64_t)si * g.k_inner + (int64_t)h * 64;
  if (PRE) {
    const __nv_bfloat16* qb = reinterpret_cast<const __nv_bfloat16*>(q_) + qoff;
    const __nv_bfloat16* kb = reinterpret_cast<const __nv_bfloat16*>(kv_) + koff;
#pragma unroll
    for (int i = 0; i < NMAX; ++i) {
      xq[i] = xk[i] = xv[i] = make_float2(0.f, 0.f);
      if (i < n) {
        xq[i] = __bfloat1622float2(reinterpret_cast<const __nv_bfloat162*>(qb + (int64_t)i * g.q_tok)[lane]);
        xk[i] = __bfloat1622float2(reinterpret_cast<const __nv_bfloat162*>(kb + (int64_t)i * g.k_tok)[lane]);
        xv[i] = __bfloat1622float2(reinterpret_cast<const __nv_bfloat162*>(kb + (int64_t)i * g.k_tok + I)[lane]);
      }
    }
  } else {
    const float* qb = reinterpret_cast<const float*>(q_) + qoff;
    const float* kb = reinterpret_cast<const float*>(kv_) + koff;
    const float2 qs = reinterpret_cast<const float2*>(q_scale)[lane], ks = reinterpret_cast<const float2*>(k_scale)[lane];
#pragma unroll
    for (int i = 0; i < NMAX; ++i) {
      xq[i] = xk[i] = xv[i] = make_float2(0.f, 0.f);
      if (i < n) {
        xq[i] = reinterpret_cast<const float2*>(qb + (int64_t)i * g.q_tok)[lane];
        xk[i] = reinterpret_cast<const float2*>(kb + (int64_t)i * g.k_tok)[lane];
        xv[i] = reinterpret_cast<const float2*>(kb + (int64_t)i * g.k_tok + I)[lane];
      }
    }
    // F.normalize(q), F.normalize(k) then * q_scale / k_scale (attention.py:153-155)
#pragma unroll
    for (int i = 0; i < NMAX; ++i) {
      if (i < n) {
        // 1 / max(||x||, 1e-12) as one rsqrt per token (the kernel is instruction-bound: ~2.8 k instructions per warp
        // with IEEE sqrt / divide / expf, profiles/r01_small_kernels_ncu.txt); the fixed scale 8 is folded into q
        const float iq = rsqrtf(fmaxf(warp_sum(xq[i].x * xq[i].x + xq[i].y * xq[i].y), 1e-24f)) * g.scale;
        const float ik = rsqrtf(fmaxf(warp_sum(xk[i].x * xk[i].x + xk[i].y * xk[i].y), 1e-24f));
        xq[i].x = (xq[i].x * iq) * qs.x; xq[i].y = (xq[i].y * iq) * qs.y;
        xk[i].x = (xk[i].x * ik) * ks.x; xk[i].y = (xk[i].y * ik) * ks.y;
      }
    }
  }
  const float slope = (g.causal && alibi_slopes) ? alibi_slopes[h] : 0.f;
  const int64_t ob = (int64_t)so * g.o_outer + (int64_t)si * g.o_inner + (int64_t)h * 64;
#pragma unroll
  for (int i = 0; i < NMAX; ++i) {
    if (i < n) {
      float sc[NMAX];
      float m = -FLT_MAX;
#pragma unroll
      for (int j = 0; j < NMAX; ++j) {
        sc[j] = -FLT_MAX;
        if (j < n && (!g.causal || j <= i)) {
          float a = warp_sum(fmaf(xq[i].x, xk[j].x, xq[i].y * xk[j].y));             // identical in every lane
          if (g.causal) a += -fabsf((float)(j - i)) * slope;                           // ALiBi (attention.py:214-227)
          sc[j] = a;
          m = fmaxf(m, a);
        }
      }
      float sum = 0.f;
      float2 o = make_float2(0.f, 0.f);
#pragma unroll
      for (int j = 0; j < NMAX; ++j) {
        if (j < n && (!g.causal || j <= i)) {
          const float e = __expf(sc[j] - m);
          sum += e;
          o.x = fmaf(e, xv[j].x, o.x);
          o.y = fmaf(e, xv[j].y, o.y);
        }
      }
      const float inv = __fdividef(1.f, sum);
      const int64_t off = ob + (int64_t)i * g.o_tok;
      if (g.out_bf16) reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(out) + off)[lane] = pack_bf16x2(o.x * inv, o.y * inv);
      else reinterpret_cast<float2*>(reinterpret_cast<float*>(out) + off)[lane] = make_float2(o.x * inv, o.y * inv);
    }
  }
}


// ------------------------------------------------------------------------------------------
// Temporal attention on pre-normalised bf16 operands with warp-level tensor-core MMAs (mma.sync m16n8k16): one warp per
// (sequence, head), n <= 16 tokens.  The shuffle kernel above spends ~2.8 k instructions per warp on 45 dot products
// reduced across lanes; here S = Q K^T is 8 MMAs, P V another 8, and the softmax runs on the accumulator fragments
// (rows live in lane quads).  Q / K / V rows (128 B each) are staged in shared memory with 16-byte loads (row stride
// 144 B: conflict-free ldmatrix), rows >= n are zero.  [not compiled for the CPU executor: PHK_CUDA_EMU]
// ------------------------------------------------------------------------------------------
#ifndef PHK_CUDA_EMU
constexpr int MMA_WARPS = 4, MMA_LD = 72;  // 4 x 3 x 16 x 144 B = 27 KB static shared memory  // bf16 elements per staged row (64 + 8 pad)

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(MMA_WARPS * 32) attention_small_mma_kernel(const __nv_bfloat16* __restrict__ q,
                                                                            const __nv_bfloat16* __restrict__ kv,
                                                                            const float* __restrict__ alibi_slopes,
                                                                            __nv_bfloat16* __restrict__ out, phk_attn_geom_t g) {
  pdl_prologue();
  __shared__ __align__(16) __nv_bfloat16 sm[MMA_WARPS][3][16][MMA_LD];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t pair = (int64_t)blockIdx.x * MMA_WARPS + w;
  const int64_t npairs = (int64_t)g.n_outer * g.n_inner * g.heads;
  if (pair >= npairs) return;  // whole warp exits together (no block-wide barrier below)
  const int h = (int)(pair % g.heads);
  const int seq = (int)(pair / g.heads);
  const int so = seq / g.n_inner, si = seq - so * g.n_inner;
  const int n = g.n_q, I = g.heads * 64;
  const __nv_bfloat16* qb = q + (int64_t)so * g.q_outer + (int64_t)si * g.q_inner + (int64_t)h * 64;
  const __nv_bfloat16* kb = kv + (int64_t)so * g.k_outer + (int64_t)si * g.k_inner + (int64_t)h * 64;
  __nv_bfloat16 (*sQ)[MMA_LD] = sm[w][0];
  __nv_bfloat16 (*sK)[MMA_LD] = sm[w][1];
  __nv_bfloat16 (*sV)[MMA_LD] = sm[w][2];
  // stage: 3 operands x 16 rows x 8 chunks of 16 B = 384 chunks, 12 per lane; rows >= n are zero
#pragma unroll
  for (int it = 0; it < 12; ++it) {
    const int idx = it * 32 + lane;
    const int op = idx >> 7, row = (idx >> 3) & 15, ch = idx & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (row < n) {
      const __nv_bfloat16* src = op == 0 ? qb + (int64_t)row * g.q_tok : kb + (int64_t)row * g.k_tok + (op == 2 ? I : 0);
      v = *reinterpret_cast<const uint4*>(src + ch * 8);
    }
    *reinterpret_cast<uint4*>(&sm[w][op][row][ch * 8]) = v;
  }
  __syncwarp();
  const int gq = lane >> 2, t = lane & 3;
  // S[16 x 16] = Q K^T: two key tiles of 8, four k-steps of 16 dims
  float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    uint32_t a[4], b[4];
    ldmatrix_x4(a, &sQ[(lane & 7) + 8 * ((lane >> 3) & 1)][ks * 16 + 8 * (lane >> 4)]);
    ldmatrix_x4(b, &sK[(lane & 7) + 8 * (lane >> 4)][ks * 16 + 8 * ((lane >> 3) & 1)]);
    mma_bf16_16816(s0, a, b[0], b[1]);  // keys 0..7
    mma_bf16_16816(s1, a, b[2], b[3]);  // keys 8..15
  }
  // softmax over the 16 keys of rows gq (c0, c1) and gq + 8 (c2, c3); key of element e of tile tl: tl * 8 + 2 t + e
  const float slope = (g.causal && alibi_slopes) ? alibi_slopes[h] : 0.f;
  float p[2][4];  // [key tile][c0..c3]
#pragma unroll
  for (int tl = 0; tl < 2; ++tl)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int row = gq + 8 * (e >> 1), key = tl * 8 + 2 * t + (e & 1);
      float v = tl == 0 ? s0[e] : s1[e];
      if (g.causal) v += -fabsf((float)(key - row)) * slope;  // ALiBi (attention.py:214-227)
      const bool ok = key < n && (!g.causal || key <= row);
      p[tl][e] = ok ? v : -FLT_MAX;
    }
  float inv[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {  // r = 0: row gq, r = 1: row gq + 8
    float m = fmaxf(fmaxf(p[0][2 * r], p[0][2 * r + 1]), fmaxf(p[1][2 * r], p[1][2 * r + 1]));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    float sum = 0.f;
#pragma unroll
    for (int tl = 0; tl < 2; ++tl)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float v = p[tl][2 * r + e];
        const float ex = v == -FLT_MAX ? 0.f : __expf(v - m);
        p[tl][2 * r + e] = ex;
        sum += ex;
      }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    inv[r] = sum > 0.f ? __fdividef(1.f, sum) : 0.f;  // (rows >= n: all keys masked, never stored)
  }
  // P as the A operand of P V (16 x 16, k = keys): the accumulator layout of S IS the A-fragment layout
  uint32_t pa[4];
  pa[0] = pack_bf16x2(p[0][0], p[0][1]);  // row gq,     keys 2t, 2t+1
  pa[1] = pack_bf16x2(p[0][2], p[0][3]);  // row gq + 8, keys 2t, 2t+1
  pa[2] = pack_bf16x2(p[1][0], p[1][1]);  // row gq,     keys 8 + 2t, ..
  pa[3] = pack_bf16x2(p[1][2], p[1][3]);  // row gq + 8, keys 8 + 2t, ..
  const int64_t ob = (int64_t)so * g.o_outer + (int64_t)si * g.o_inner + (int64_t)h * 64;
#pragma unroll
  for (int dp = 0; dp < 4; ++dp) {  // two 8-dim tiles per ldmatrix.x4.trans
    uint32_t b[4];
    ldmatrix_x4_trans(b, &sV[(lane & 7) + 8 * ((lane >> 3) & 1)][(2 * dp + (lane >> 4)) * 8]);
    float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
    mma_bf16_16816(o0, pa, b[0], b[1]);  // dims (2 dp) * 8 ..
    mma_bf16_16816(o1, pa, b[2], b[3]);  // dims (2 dp + 1) * 8 ..
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = gq + 8 * r;
      if (row < n) {
        __nv_bfloat16* orow = out + ob + (int64_t)row * g.o_tok;
        *reinterpret_cast<uint32_t*>(orow + (2 * dp) * 8 + 2 * t) = pack_bf16x2(o0[2 * r] * inv[r], o0[2 * r + 1] * inv[r]);
        *reinterpret_cast<uint32_t*>(orow + (2 * dp + 1) * 8 + 2 * t) = pack_bf16x2(o1[2 * r] * inv[r], o1[2 * r + 1] * inv[r]);
      }
    }
  }
}
#endif  // PHK_CUDA_EMU


// ------------------------------------------------------------------------------------------
// Self-attention of short sequences (16 < n <= 64: the spatial transformer's 8 x 8 token frames) on the pre-normalised
// token-major bf16 operands, warp-level MMAs: one CTA of four warps per (sequence, head), every warp owns 16 query rows.
// The wgmma kernel (attention_tc_kernel) spends its life in prologue / barrier round trips at this size -- one 64-key
// chunk, half of its 128-row tile empty, 576 CTAs on 296 resident slots = two rounds (8.9 us at 72 x 64 x 8 heads);
// here 576 CTAs of 128 threads and 27 KB are resident at once and a CTA is a 24 KB copy + 64 MMAs per warp.
// Position bias fp32 [heads, n, n] or NULL; no masks, not causal (those take phk_attention).  [not on the CPU executor]
// ------------------------------------------------------------------------------------------
#ifndef PHK_CUDA_EMU
constexpr int MID_N = 64;

__global__ void __launch_bounds__(128) attention_mid_mma_kernel(const __nv_bfloat16* __restrict__ Qn, int64_t ld_q,
                                                                const __nv_bfloat16* __restrict__ KVn, int64_t ld_kv,
                                                                const float* __restrict__ bias,
                                                                __nv_bfloat16* __restrict__ out, int64_t ld_o, int n,
                                                                int heads) {
  pdl_prologue();
  __shared__ __align__(16) __nv_bfloat16 sm[3][MID_N][MMA_LD];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int h = blockIdx.x, seq = blockIdx.y;
  const int I = heads * 64;
  const __nv_bfloat16* qb = Qn + (int64_t)seq * n * ld_q + (int64_t)h * 64;
  const __nv_bfloat16* kb = KVn + (int64_t)seq * n * ld_kv + (int64_t)h * 64;
  // stage: 3 operands x 64 rows x 8 chunks of 16 B = 1536 chunks, 12 per thread; rows >= n are zero
#pragma unroll
  for (int it = 0; it < 12; ++it) {
    const int idx = it * 128 + threadIdx.x;
    const int op = idx >> 9, row = (idx >> 3) & 63, ch = idx & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (row < n) {
      const __nv_bfloat16* src = op == 0 ? qb + (int64_t)row * ld_q : kb + (int64_t)row * ld_kv + (op == 2 ? I : 0);
      v = *reinterpret_cast<const uint4*>(src + ch * 8);
    }
    *reinterpret_cast<uint4*>(&sm[op][row][ch * 8]) = v;
  }
  __syncthreads();
  const int r0 = w * 16;
  if (r0 >= n) return;
  __nv_bfloat16 (*sQ)[MMA_LD] = sm[0];
  __nv_bfloat16 (*sK)[MMA_LD] = sm[1];
  __nv_bfloat16 (*sV)[MMA_LD] = sm[2];
  const int gq = lane >> 2, t = lane & 3;
  uint32_t a[4][4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) ldmatrix_x4(a[ks], &sQ[r0 + (lane & 7) + 8 * ((lane >> 3) & 1)][ks * 16 + 8 * (lane >> 4)]);
  // S[16 x 64] = Q K^T: eight key tiles of 8, four k-steps of 16 dims
  float sc[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) sc[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b[4];
      ldmatrix_x4(b, &sK[(lane & 7) + 8 * (lane >> 4) + 16 * np][ks * 16 + 8 * ((lane >> 3) & 1)]);
      mma_bf16_16816(sc[2 * np], a[ks], b[0], b[1]);
      mma_bf16_16816(sc[2 * np + 1], a[ks], b[2], b[3]);
    }
  // + position bias, padding keys masked; element e of tile nt: row r0 + gq + 8 (e >> 1), key nt * 8 + 2 t + (e & 1)
  const bool bias_vec = bias && (n % 2 == 0) && ((reinterpret_cast<uintptr_t>(bias) & 7) == 0);
  float inv[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r0 + gq + 8 * r;
    const float* brow = (bias && row < n) ? bias + ((int64_t)h * n + row) * n : nullptr;
    float m = -FLT_MAX;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = nt * 8 + 2 * t;
      float b0 = 0.f, b1 = 0.f;
      if (brow) {
        if (bias_vec && key + 1 < n) { const float2 bb = __ldg(reinterpret_cast<const float2*>(brow + key)); b0 = bb.x; b1 = bb.y; }
        else { if (key < n) b0 = __ldg(brow + key); if (key + 1 < n) b1 = __ldg(brow + key + 1); }
      }
      const float v0 = key < n ? sc[nt][2 * r] + b0 : -FLT_MAX, v1 = key + 1 < n ? sc[nt][2 * r + 1] + b1 : -FLT_MAX;
      sc[nt][2 * r] = v0; sc[nt][2 * r + 1] = v1;
      m = fmaxf(m, fmaxf(v0, v1));
    }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    float sum = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float v = sc[nt][2 * r + e];
        const float ex = v == -FLT_MAX ? 0.f : __expf(v - m);
        sc[nt][2 * r + e] = ex;
        sum += ex;
      }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    inv[r] = sum > 0.f ? __fdividef(1.f, sum) : 0.f;
  }
  uint32_t pa[4][4];  // P as the A operand of P V: four k-steps of 16 keys (the accumulator layout of S IS the A layout)
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    pa[kk][0] = pack_bf16x2(sc[2 * kk][0], sc[2 * kk][1]);
    pa[kk][1] = pack_bf16x2(sc[2 * kk][2], sc[2 * kk][3]);
    pa[kk][2] = pack_bf16x2(sc[2 * kk + 1][0], sc[2 * kk + 1][1]);
    pa[kk][3] = pack_bf16x2(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
  }
  __nv_bfloat16* obase = out + (int64_t)seq * n * ld_o + (int64_t)h * 64;
#pragma unroll
  for (int dp = 0; dp < 4; ++dp) {
    float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t b[4];
      ldmatrix_x4_trans(b, &sV[(lane & 7) + 8 * ((lane >> 3) & 1) + 16 * kk][(2 * dp + (lane >> 4)) * 8]);
      mma_bf16_16816(o0, pa[kk], b[0], b[1]);
      mma_bf16_16816(o1, pa[kk], b[2], b[3]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = r0 + gq + 8 * r;
      if (row < n) {
        __nv_bfloat16* orow = obase + (int64_t)row * ld_o;
        *reinterpret_cast<uint32_t*>(orow + (2 * dp) * 8 + 2 * t) = pack_bf16x2(o0[2 * r] * inv[r], o0[2 * r + 1] * inv[r]);
        *reinterpret_cast<uint32_t*>(orow + (2 * dp + 1) * 8 + 2 * t) = pack_bf16x2(o1[2 * r] * inv[r], o1[2 * r + 1] * inv[r]);
      }
    }
  }
}
#endif  // PHK_CUDA_EMU


// ------------------------------------------------------------------------------------------
// Cross-attention over a short text context (null-kv + L <= 32 keys, dim_head 64, bf16 output: the bf16 mode of
// MaskGit / TokenCritic, attention.py:137-181) on warp-level tensor-core MMAs.  CTA = 128 queries of one (sequence,
// head): the keys are l2-normalised, scaled and converted once per CTA into shared memory (like attention_fewkeys_kernel),
// every warp owns 16 queries: it loads their fp32 rows straight into A-fragment order (float2 per lane), normalises them
// with quad shuffles, S = Q K^T is 16 mma.sync.m16n8k16, the softmax runs on the accumulator fragments, P V another 16.
// attention_fewkeys_kernel (one thread per query, broadcast reads) needs ~5x the issue slots; it remains the path for
// fp32 output, other head sizes and the CPU executor.  [not compiled for the CPU executor: PHK_CUDA_EMU]
// ------------------------------------------------------------------------------------------
#ifndef PHK_CUDA_EMU
constexpr int XK = 32;  // key slots (null-kv + text), XK / 8 score tiles per warp

__global__ void __launch_bounds__(256) attention_cross_mma_kernel(const float* __restrict__ q, const float* __restrict__ kv,
                                                                  const float* __restrict__ null_kv,
                                                                  const float* __restrict__ q_scale,
                                                                  const float* __restrict__ k_scale,
                                                                  const uint8_t* __restrict__ key_mask,
                                                                  __nv_bfloat16* __restrict__ out, phk_attn_geom_t g) {
  pdl_prologue();
  __shared__ __align__(16) __nv_bfloat16 sK[XK][MMA_LD];
  __shared__ __align__(16) __nv_bfloat16 sV[XK][MMA_LD];
  __shared__ float s_dead[XK];  // 0: live key, 1: masked / padding
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int h = blockIdx.y, seq = blockIdx.z;
  const int so = seq / g.n_inner, si = seq - so * g.n_inner;
  const int I = g.heads * 64, nnull = g.num_null_kv, nk_all = g.n_k + nnull;
  const int kv_so = g.kv_outer_mod > 0 ? so % g.kv_outer_mod : so;
  const int mask_row = g.mask_outer_mod > 0 ? so % g.mask_outer_mod : so;
  const bool mask_dropped = g.mask_off_from >= 0 && so >= g.mask_off_from;
  // null half of a CFG pair: every text key is masked and contributes exp(-FLT_MAX - m) = 0 exactly -> only the null keys
  const int nk = (mask_dropped && key_mask) ? nnull : nk_all;
  const float* kbase = kv + (int64_t)kv_so * g.k_outer + (int64_t)si * g.k_inner + (int64_t)h * 64;
  for (int j = w; j < XK; j += 8) {  // warp per key slot: l2-normalise * k_scale -> bf16; value -> bf16; zero padding
    float2 kx = make_float2(0.f, 0.f), vx = make_float2(0.f, 0.f);
    bool dead = true;
    if (j < nk) {
      const float* kp;
      const float* vp;
      if (j < nnull) { kp = null_kv + ((int64_t)h * 2 * nnull + 2 * j) * 64; vp = kp + 64; }   // 'h (n r) d' (:148)
      else { kp = kbase + (int64_t)(j - nnull) * g.k_tok; vp = kp + I; }
      kx = reinterpret_cast<const float2*>(kp)[lane];
      vx = reinterpret_cast<const float2*>(vp)[lane];
      const float inv = 1.0f / fmaxf(sqrtf(warp_sum(kx.x * kx.x + kx.y * kx.y)), 1e-12f);
      const float2 ks = reinterpret_cast<const float2*>(k_scale)[lane];
      kx.x = (kx.x * inv) * ks.x; kx.y = (kx.y * inv) * ks.y;
      const int kj = j - nnull;
      dead = key_mask && kj >= 0 && (mask_dropped || !key_mask[(int64_t)mask_row * g.n_k + kj]);
    }
    reinterpret_cast<uint32_t*>(&sK[j][0])[lane] = pack_bf16x2(kx.x, kx.y);
    reinterpret_cast<uint32_t*>(&sV[j][0])[lane] = pack_bf16x2(vx.x, vx.y);
    if (lane == 0) s_dead[j] = dead ? 1.f : 0.f;
  }
  __syncthreads();
  const int gq = lane >> 2, t = lane & 3;
  const int r0 = blockIdx.x * 128 + w * 16;  // this warp's 16 queries
  if (r0 >= g.n_q) return;
  const float* qbase = q + (int64_t)so * g.q_outer + (int64_t)si * g.q_inner + (int64_t)h * 64;
  // A fragments of the normalised queries: lane (gq, t) holds rows gq / gq + 8, columns ks*16 + {2t, 2t+1, 2t+8, 2t+9}
  float2 qa[4][4];
  float ss0 = 0.f, ss1 = 0.f;
  const bool v0 = r0 + gq < g.n_q, v1 = r0 + gq + 8 < g.n_q;
  const float* q0p = qbase + (int64_t)(r0 + gq) * g.q_tok;
  const float* q1p = qbase + (int64_t)(r0 + gq + 8) * g.q_tok;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const int c = ks * 16 + 2 * t;
    qa[ks][0] = v0 ? *reinterpret_cast<const float2*>(q0p + c) : make_float2(0.f, 0.f);
    qa[ks][1] = v1 ? *reinterpret_cast<const float2*>(q1p + c) : make_float2(0.f, 0.f);
    qa[ks][2] = v0 ? *reinterpret_cast<const float2*>(q0p + c + 8) : make_float2(0.f, 0.f);
    qa[ks][3] = v1 ? *reinterpret_cast<const float2*>(q1p + c + 8) : make_float2(0.f, 0.f);
    ss0 += qa[ks][0].x * qa[ks][0].x + qa[ks][0].y * qa[ks][0].y + qa[ks][2].x * qa[ks][2].x + qa[ks][2].y * qa[ks][2].y;
    ss1 += qa[ks][1].x * qa[ks][1].x + qa[ks][1].y * qa[ks][1].y + qa[ks][3].x * qa[ks][3].x + qa[ks][3].y * qa[ks][3].y;
  }
  ss0 += __shfl_xor_sync(0xffffffffu, ss0, 1); ss0 += __shfl_xor_sync(0xffffffffu, ss0, 2);
  ss1 += __shfl_xor_sync(0xffffffffu, ss1, 1); ss1 += __shfl_xor_sync(0xffffffffu, ss1, 2);
  const float i0 = g.scale / fmaxf(sqrtf(ss0), 1e-12f), i1 = g.scale / fmaxf(sqrtf(ss1), 1e-12f);
  uint32_t a[4][4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const int c = ks * 16 + 2 * t;
    const float2 s_lo = *reinterpret_cast<const float2*>(q_scale + c), s_hi = *reinterpret_cast<const float2*>(q_scale + c + 8);
    a[ks][0] = pack_bf16x2(qa[ks][0].x * i0 * s_lo.x, qa[ks][0].y * i0 * s_lo.y);
    a[ks][1] = pack_bf16x2(qa[ks][1].x * i1 * s_lo.x, qa[ks][1].y * i1 * s_lo.y);
    a[ks][2] = pack_bf16x2(qa[ks][2].x * i0 * s_hi.x, qa[ks][2].y * i0 * s_hi.y);
    a[ks][3] = pack_bf16x2(qa[ks][3].x * i1 * s_hi.x, qa[ks][3].y * i1 * s_hi.y);
  }
  // S[16 x 32] = Q K^T: four key tiles of 8, four k-steps of 16 dims
  float sc[4][4];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) sc[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t b[4];
      ldmatrix_x4(b, &sK[(lane & 7) + 8 * (lane >> 4) + 16 * np][ks * 16 + 8 * ((lane >> 3) & 1)]);
      mma_bf16_16816(sc[2 * np], a[ks], b[0], b[1]);
      mma_bf16_16816(sc[2 * np + 1], a[ks], b[2], b[3]);
    }
  // softmax over the key slots; masked / padding keys: the reference fills -finfo.max (:168) -> weight exactly 0 next to
  // the always-live null keys (the dispatcher only takes this kernel when num_null_kv > 0)
  float inv[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float m = -FLT_MAX;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = nt * 8 + 2 * t + e;
        if (s_dead[key] != 0.f) sc[nt][2 * r + e] = -FLT_MAX;
        m = fmaxf(m, sc[nt][2 * r + e]);
      }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    float sum = 0.f;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float v = sc[nt][2 * r + e];
        const float ex = v == -FLT_MAX ? 0.f : __expf(v - m);
        sc[nt][2 * r + e] = ex;
        sum += ex;
      }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    inv[r] = sum > 0.f ? __fdividef(1.f, sum) : 0.f;
  }
  uint32_t pa[2][4];  // P as the A operand of P V, two k-steps of 16 keys
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) {
    pa[kk][0] = pack_bf16x2(sc[2 * kk][0], sc[2 * kk][1]);
    pa[kk][1] = pack_bf16x2(sc[2 * kk][2], sc[2 * kk][3]);
    pa[kk][2] = pack_bf16x2(sc[2 * kk + 1][0], sc[2 * kk + 1][1]);
    pa[kk][3] = pack_bf16x2(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
  }
  const int64_t ob = (int64_t)so * g.o_outer + (int64_t)si * g.o_inner + (int64_t)h * 64;
#pragma unroll
  for (int dp = 0; dp < 4; ++dp) {
    float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      uint32_t b[4];
      ldmatrix_x4_trans(b, &sV[(lane & 7) + 8 * ((lane >> 3) & 1) + 16 * kk][(2 * dp + (lane >> 4)) * 8]);
      mma_bf16_16816(o0, pa[kk], b[0], b[1]);
      mma_bf16_16816(o1, pa[kk], b[2], b[3]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = r0 + gq + 8 * r;
      if (row < g.n_q) {
        __nv_bfloat16* orow = out + ob + (int64_t)row * g.o_tok;
        *reinterpret_cast<uint32_t*>(orow + (2 * dp) * 8 + 2 * t) = pack_bf16x2(o0[2 * r] * inv[r], o0[2 * r + 1] * inv[r]);
        *reinterpret_cast<uint32_t*>(orow + (2 * dp + 1) * 8 + 2 * t) = pack_bf16x2(o1[2 * r] * inv[r], o1[2 * r + 1] * inv[r]);
      }
    }
  }
}
#endif  // PHK_CUDA_EMU

// ------------------------------------------------------------------------------------------
// The same cross-attention on PACKED operands.  The keys / values of a sample do not change over its demasking iterations
// nor between the query tiles of an iteration, yet attention_cross_mma_kernel re-normalised them in every CTA (one extra
// dependent global-load latency + 32 warp reductions per CTA).  cross_kv_pack_kernel does it once per transformer call for
// all layers: pack[(l * ctx_b + b) * heads + h] = { K^ [32 slots][64] bf16 (l2-normalised * k_scale; null keys first, zero
// padding), V [32][64] bf16 }, dead[(l * ctx_b + b)][32] (1: masked text key or padding).  The queries arrive as the bf16
// operand phk_gemm_bf16_qnorm writes (normalised, scaled), so the attention CTA only copies 8 KB, loads its A fragments
// and runs the 32 MMAs.  [not compiled for the CPU executor]
// ------------------------------------------------------------------------------------------
#ifndef PHK_CUDA_EMU
struct CrossPackLayer { const float* kv; const float* null_kv; const float* k_scale; };
struct CrossPackArgs { CrossPackLayer layer[16]; };

__global__ void __launch_bounds__(256) cross_kv_pack_kernel(CrossPackArgs a, const uint8_t* __restrict__ key_mask,
                                                            __nv_bfloat16* __restrict__ pack, float* __restrict__ dead,
                                                            int depth, int ctx_b, int L, int heads, int nnull) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int64_t total = (int64_t)depth * ctx_b * heads * XK;
  if (warp >= total) return;
  const int j = (int)(warp % XK);
  const int h = (int)((warp / XK) % heads);
  const int b = (int)((warp / ((int64_t)XK * heads)) % ctx_b);
  const int l = (int)(warp / ((int64_t)XK * heads * ctx_b));
  const CrossPackLayer& ly = a.layer[l];
  const int I = heads * 64;
  float2 kx = make_float2(0.f, 0.f), vx = make_float2(0.f, 0.f);
  bool is_dead = true;
  if (j < nnull + L) {
    const float* kp;
    const float* vp;
    if (j < nnull) { kp = ly.null_kv + ((int64_t)h * 2 * nnull + 2 * j) * 64; vp = kp + 64; }   // 'h (n r) d' (:148)
    else { kp = ly.kv + ((int64_t)b * L + (j - nnull)) * 2 * I + (int64_t)h * 64; vp = kp + I; }
    kx = reinterpret_cast<const float2*>(kp)[lane];
    vx = reinterpret_cast<const float2*>(vp)[lane];
    const float inv = 1.0f / fmaxf(sqrtf(warp_sum(kx.x * kx.x + kx.y * kx.y)), 1e-12f);
    const float2 ks = reinterpret_cast<const float2*>(ly.k_scale)[lane];
    kx.x = (kx.x * inv) * ks.x; kx.y = (kx.y * inv) * ks.y;
    is_dead = key_mask && j >= nnull && !key_mask[(int64_t)b * L + (j - nnull)];
  }
  __nv_bfloat16* base = pack + (((int64_t)l * ctx_b + b) * heads + h) * (2 * XK * 64);
  reinterpret_cast<uint32_t*>(base + j * 64)[lane] = pack_bf16x2(kx.x, kx.y);
  reinterpret_cast<uint32_t*>(base + XK * 64 + j * 64)[lane] = pack_bf16x2(vx.x, vx.y);
  if (h == 0 && lane == 0) dead[((int64_t)l * ctx_b + b) * XK + j] = is_dead ? 1.f : 0.f;
}

// grid (ceil(n_q / 128), heads, sequences); sequence `seq` reads the pack of text seq % ctx_b; sequences >= null_from (the
// null half of a CFG pair) see only the null keys.  Qn / out: token-major bf16 rows, sequence stride n_q rows.
__global__ void __launch_bounds__(256) attention_cross_packed_kernel(const __nv_bfloat16* __restrict__ Qn, int64_t ld_q,
                                                                     const __nv_bfloat16* __restrict__ pack,
                                                                     const float* __restrict__ dead,
                                                                     __nv_bfloat16* __restrict__ out, int64_t ld_o, int n_q,
                                                                     int heads, int ctx_b, int nnull, int null_from) {
  pdl_prologue();
  __shared__ __align__(16) __nv_bfloat16 sK[XK][MMA_LD];
  __shared__ __align__(16) __nv_bfloat16 sV[XK][MMA_LD];
  __shared__ float s_dead[XK];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int h = blockIdx.y, seq = blockIdx.z;
  const int b = seq % ctx_b;
  const bool null_half = null_from >= 0 && seq >= null_from;
  const __nv_bfloat16* pk = pack + ((int64_t)b * heads + h) * (2 * XK * 64);
  for (int i = threadIdx.x; i < 2 * XK * 8; i += 256) {  // 2 x 32 rows x 8 sixteen-byte pieces
    const int which = i / (XK * 8), r = (i / 8) % XK, c = i % 8;
    const uint4 v = reinterpret_cast<const uint4*>(pk + which * (XK * 64) + r * 64)[c];
    *reinterpret_cast<uint4*>(which ? &sV[r][c * 8] : &sK[r][c * 8]) = v;
  }
  if (threadIdx.x < XK) s_dead[threadIdx.x] = (null_half && threadIdx.x >= nnull) ? 1.f : dead[(int64_t)b * XK + threadIdx.x];
  const int gq = lane >> 2, t = lane & 3;
  const int r0 = blockIdx.x * 128 + w * 16;  // this warp's 16 queries
  // A fragments straight from the bf16 rows: lane (gq, t) holds rows gq / gq + 8, columns ks*16 + {2t, 2t+1} and + 8
  uint32_t a[4][4];
  const bool v0 = r0 + gq < n_q, v1 = r0 + gq + 8 < n_q;
  const __nv_bfloat16* q0p = Qn + ((int64_t)seq * n_q + r0 + gq) * ld_q + h * 64;
  const __nv_bfloat16* q1p = q0p + 8 * ld_q;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const int c = ks * 16 + 2 * t;
    a[ks][0] = v0 ? *reinterpret_cast<const uint32_t*>(q0p + c) : 0u;
    a[ks][1] = v1 ? *reinterpret_cast<const uint32_t*>(q1p + c) : 0u;
    a[ks][2] = v0 ? *reinterpret_cast<const uint32_t*>(q0p + c + 8) : 0u;
    a[ks][3] = v1 ? *reinterpret_cast<const uint32_t*>(q1p + c + 8) : 0u;
  }
  __syncthreads();
  if (r0 >= n_q) return;
  float sc[4][4];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) sc[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int np = 0; np < 2; ++np) {
      uint32_t bfr[4];
      ldmatrix_x4(bfr, &sK[(lane & 7) + 8 * (lane >> 4) + 16 * np][ks * 16 + 8 * ((lane >> 3) & 1)]);
      mma_bf16_16816(sc[2 * np], a[ks], bfr[0], bfr[1]);
      mma_bf16_16816(sc[2 * np + 1], a[ks], bfr[2], bfr[3]);
    }
  float inv[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float m = -FLT_MAX;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = nt * 8 + 2 * t + e;
        if (s_dead[key] != 0.f) sc[nt][2 * r + e] = -FLT_MAX;
        m = fmaxf(m, sc[nt][2 * r + e]);
      }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    float sum = 0.f;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float v = sc[nt][2 * r + e];
        const float ex = v == -FLT_MAX ? 0.f : __expf(v - m);
        sc[nt][2 * r + e] = ex;
        sum += ex;
      }
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    inv[r] = sum > 0.f ? __fdividef(1.f, sum) : 0.f;
  }
  uint32_t pa[2][4];
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) {
    pa[kk][0] = pack_bf16x2(sc[2 * kk][0], sc[2 * kk][1]);
    pa[kk][1] = pack_bf16x2(sc[2 * kk][2], sc[2 * kk][3]);
    pa[kk][2] = pack_bf16x2(sc[2 * kk + 1][0], sc[2 * kk + 1][1]);
    pa[kk][3] = pack_bf16x2(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
  }
  __nv_bfloat16* obase = out + ((int64_t)seq * n_q) * ld_o + h * 64;
#pragma unroll
  for (int dp = 0; dp < 4; ++dp) {
    float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      uint32_t bfr[4];
      ldmatrix_x4_trans(bfr, &sV[(lane & 7) + 8 * ((lane >> 3) & 1) + 16 * kk][(2 * dp + (lane >> 4)) * 8]);
      mma_bf16_16816(o0, pa[kk], bfr[0], bfr[1]);
      mma_bf16_16816(o1, pa[kk], bfr[2], bfr[3]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = r0 + gq + 8 * r;
      if (row < n_q) {
        __nv_bfloat16* orow = obase + (int64_t)row * ld_o;
        *reinterpret_cast<uint32_t*>(orow + (2 * dp) * 8 + 2 * t) = pack_bf16x2(o0[2 * r] * inv[r], o0[2 * r + 1] * inv[r]);
        *reinterpret_cast<uint32_t*>(orow + (2 * dp + 1) * 8 + 2 * t) = pack_bf16x2(o1[2 * r] * inv[r], o1[2 * r + 1] * inv[r]);
      }
    }
  }
}
#endif  // PHK_CUDA_EMU


template <int NMAX, bool PRE = false>
static int launch_attention_warp64(const void* q, const void* kv, const float* q_scale, const float* k_scale,
                                   const float* alibi_slopes, void* out, const phk_attn_geom_t& g, cudaStream_t st) {
  const int64_t npairs = (int64_t)g.n_outer * g.n_inner * g.heads;
  PHK_CUDA(launch_pdl(attention_warp64_kernel<NMAX, PRE>, dim3((unsigned)((npairs + 7) / 8)), dim3(256), (size_t)0, st, q, kv,
                      q_scale, k_scale, alibi_slopes, out, g));
  PHK_LAUNCH_CHECK();
  return 0;
}

template <int DH, int NMAX>
static int launch_attention_rows(const float* q, const float* kv, const float* q_scale, const float* k_scale,
                                 const float* alibi_slopes, void* out, const phk_attn_geom_t& g, cudaStream_t st) {
  const int n = g.n_q, G = ROWS_QUERIES / n;
  const int64_t npairs = (int64_t)g.n_outer * g.n_inner * g.heads;
  const size_t smem = (size_t)2 * G * (n * DH + 16) * sizeof(float);
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(attention_rows_kernel<DH, NMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)(2 * ROWS_QUERIES * (DH + 16) * sizeof(float))));
    mark_configured(&configured_mask);
  }
  PHK_CUDA(launch_pdl(attention_rows_kernel<DH, NMAX>, dim3((unsigned)((npairs + G - 1) / G)), dim3(ROWS_THREADS), smem, st, q,
                      kv, q_scale, k_scale, alibi_slopes, out, g));
  PHK_LAUNCH_CHECK();
  return 0;
}

template <int DH, int NMAX>
static int launch_attention_small_n(const float* q, const float* kv, const float* q_scale, const float* k_scale,
                                    const float* alibi_slopes, void* out, const phk_attn_geom_t& g, cudaStream_t st) {
  const int64_t npairs = (int64_t)g.n_outer * g.n_inner * g.heads;
  const size_t smem = (size_t)SMALL_WARPS * (2 * g.n_q * (DH + 1) + g.n_q * (g.n_q + 1)) * sizeof(float);
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(attention_small_kernel<DH, NMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)(SMALL_WARPS * (2 * SMALL_N * (DH + 1) + SMALL_N * (SMALL_N + 1)) * sizeof(float))));
    mark_configured(&configured_mask);
  }
  PHK_CUDA(launch_pdl(attention_small_kernel<DH, NMAX>, dim3((unsigned)((npairs + SMALL_WARPS - 1) / SMALL_WARPS)),
                      dim3(SMALL_WARPS * 32), smem, st, q, kv, q_scale, k_scale, alibi_slopes, out, g));
  PHK_LAUNCH_CHECK();
  return 0;
}

template <int DH>
static int launch_attention_small(const float* q, const float* kv, const float* q_scale, const float* k_scale,
                                  const float* alibi_slopes, void* out, const phk_attn_geom_t& g, cudaStream_t st) {
  const int n = g.n_q;
  const bool aligned = g.q_tok % 4 == 0 && g.q_outer % 4 == 0 && g.q_inner % 4 == 0 && g.k_tok % 4 == 0 &&
                       g.k_outer % 4 == 0 && g.k_inner % 4 == 0 && g.o_tok % 8 == 0 && g.o_outer % 8 == 0 &&
                       g.o_inner % 8 == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0 &&
                       (reinterpret_cast<uintptr_t>(kv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                       (reinterpret_cast<uintptr_t>(q_scale) & 15) == 0 && (reinterpret_cast<uintptr_t>(k_scale) & 15) == 0;
  if (aligned && DH == 64) {  // warp per (sequence, head), registers + shuffles only
    if (n <= 3) return launch_attention_warp64<3>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
    if (n <= 5) return launch_attention_warp64<5>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
    if (n <= 9) return launch_attention_warp64<9>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
    if (n <= 12) return launch_attention_warp64<12>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
    return launch_attention_warp64<16>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
  }
  if (aligned) {  // thread-per-query kernel
    if (n <= 3) return launch_attention_rows<DH, 3>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
    if (n <= 5) return launch_attention_rows<DH, 5>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
    if (n <= 9) return launch_attention_rows<DH, 9>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
    if (n <= 12) return launch_attention_rows<DH, 12>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
    return launch_attention_rows<DH, 16>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
  }
  if (n <= 3) return launch_attention_small_n<DH, 3>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
  if (n <= 5) return launch_attention_small_n<DH, 5>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
  if (n <= 9) return launch_attention_small_n<DH, 9>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
  if (n <= 12) return launch_attention_small_n<DH, 12>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
  return launch_attention_small_n<DH, 16>(q, kv, q_scale, k_scale, alibi_slopes, out, g, st);
}

template <int DH>
static int launch_attention(const float* q, const float* kv, const float* null_kv, const float* q_scale,
                            const float* k_scale, const float* bias, const uint8_t* key_mask,
                            const float* alibi_slopes, void* out, const phk_attn_geom_t& g, cudaStream_t st) {
  const size_t smem = sizeof(AttSmem<DH>);
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(attention_kernel<DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mark_configured(&configured_mask);
  }
  dim3 grid((unsigned)((g.n_q + TQ - 1) / TQ), (unsigned)g.heads, (unsigned)(g.n_outer * g.n_inner));
  PHK_CUDA(launch_pdl(attention_kernel<DH>, dim3(grid), dim3(ATT_THREADS), (size_t)(smem), st, q, kv, null_kv, q_scale, k_scale, bias, key_mask, alibi_slopes, out, g));
  PHK_LAUNCH_CHECK();
  return 0;
}

}  // namespace phk

using namespace phk;

extern "C" int phk_attention(const float* q, const float* kv, const float* null_kv, const float* q_scale,
                             const float* k_scale, const float* bias, const uint8_t* key_mask,
                             const float* alibi_slopes, void* out, const phk_attn_geom_t* g, phk_stream_t s) {
  Prof prof_(FAM_ATTENTION, s, g ? 4.0 * (double)g->n_outer * g->n_inner * g->heads * g->n_q * (g->n_k + g->num_null_kv) * g->dim_head : 0.0);
  PHK_REQUIRE(q && kv && q_scale && k_scale && out && g, PHK_E_ARG, "phk_attention: null pointer");
  PHK_REQUIRE(g->n_outer > 0 && g->n_inner > 0 && g->n_q > 0 && g->n_k >= 0 && g->heads > 0, PHK_E_ARG,
              "phk_attention: bad geometry");
  PHK_REQUIRE(g->num_null_kv == 0 || null_kv, PHK_E_ARG, "phk_attention: null_kv missing");
  PHK_REQUIRE(g->n_k + g->num_null_kv > 0, PHK_E_SHAPE, "phk_attention: no keys");
  PHK_REQUIRE(!g->causal || (g->num_null_kv == 0 && alibi_slopes), PHK_E_UNSUPPORTED,
              "phk_attention: causal attention takes ALiBi slopes and no null-kv (attention.py:109-110,303)");
  PHK_REQUIRE((int64_t)g->n_outer * g->n_inner <= 65535 * 1 || true, PHK_E_UNSUPPORTED, "");
  PHK_REQUIRE((int64_t)g->n_outer * g->n_inner <= 2147483647LL && g->heads <= 65535, PHK_E_UNSUPPORTED,
              "phk_attention: grid too large");
  cudaStream_t st = to_stream(s);
  // gridDim.z is limited to 65535: fold sequences if needed
  PHK_REQUIRE((int64_t)g->n_outer * g->n_inner <= 65535, PHK_E_UNSUPPORTED, "phk_attention: more than 65535 sequences");
  if (g->n_q == g->n_k && g->n_k <= SMALL_N && g->num_null_kv == 0 && !bias && !key_mask &&
      (g->dim_head == 64 || g->dim_head == 32)) {
    if (g->dim_head == 64) return launch_attention_small<64>(q, kv, q_scale, k_scale, alibi_slopes, out, *g, st);
    return launch_attention_small<32>(q, kv, q_scale, k_scale, alibi_slopes, out, *g, st);
  }
#ifndef PHK_CUDA_EMU
  {  // bf16-mode cross-attention over <= 32 key slots on warp-level MMAs
    if (!g->causal && !bias && g->out_bf16 && g->dim_head == 64 && g->num_null_kv > 0 &&
        g->n_k + g->num_null_kv <= XK && g->q_tok % 2 == 0 && g->q_outer % 2 == 0 && g->q_inner % 2 == 0 && g->k_tok % 2 == 0 &&
        g->k_outer % 2 == 0 && g->k_inner % 2 == 0 && g->o_tok % 2 == 0 && g->o_outer % 2 == 0 && g->o_inner % 2 == 0 &&
        ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(kv) | reinterpret_cast<uintptr_t>(null_kv) |
          reinterpret_cast<uintptr_t>(q_scale) | reinterpret_cast<uintptr_t>(k_scale)) & 7) == 0 &&
        (reinterpret_cast<uintptr_t>(out) & 3) == 0) {
      dim3 grid((unsigned)((g->n_q + 127) / 128), (unsigned)g->heads, (unsigned)(g->n_outer * g->n_inner));
      PHK_CUDA(launch_pdl(attention_cross_mma_kernel, grid, dim3(256), (size_t)0, st, q, kv, null_kv, q_scale, k_scale, key_mask,
                          (__nv_bfloat16*)out, *g));
      PHK_LAUNCH_CHECK();
      return 0;
    }
  }
#endif
  if (!g->causal && !bias && g->n_k + g->num_null_kv <= FEW_KEYS && (g->dim_head == 64 || g->dim_head == 32) &&
      g->q_tok % 4 == 0 && g->q_outer % 4 == 0 && g->q_inner % 4 == 0 && g->o_tok % 8 == 0 && g->o_outer % 8 == 0 &&
      g->o_inner % 8 == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    if (g->dim_head == 64) return launch_attention_fewkeys<64>(q, kv, null_kv, q_scale, k_scale, key_mask, out, *g, st);
    return launch_attention_fewkeys<32>(q, kv, null_kv, q_scale, k_scale, key_mask, out, *g, st);
  }
  switch (g->dim_head) {
    case 16: return launch_attention<16>(q, kv, null_kv, q_scale, k_scale, bias, key_mask, alibi_slopes, out, *g, st);
    case 32: return launch_attention<32>(q, kv, null_kv, q_scale, k_scale, bias, key_mask, alibi_slopes, out, *g, st);
    case 64: return launch_attention<64>(q, kv, null_kv, q_scale, k_scale, bias, key_mask, alibi_slopes, out, *g, st);
    case 128: return launch_attention<128>(q, kv, null_kv, q_scale, k_scale, bias, key_mask, alibi_slopes, out, *g, st);
    default: PHK_REQUIRE(false, PHK_E_UNSUPPORTED, "phk_attention: dim_head must be 16, 32, 64 or 128");
  }
  return 0;
}

// Small-sequence self-attention (n <= 16, dim_head 64: the temporal transformer, n = T') on the bf16 operands that
// phk_gemm_bf16_qkv writes: Qn / KVn already l2-normalised and scaled (similarity scale folded into q), addressed
// through the same geometry (strides in ELEMENTS).  No null-kv, bias or key mask; causal takes ALiBi slopes.
extern "C" int phk_attention_small_bf16(const void* Qn, const void* KVn, const float* alibi_slopes, void* out,
                                        const phk_attn_geom_t* g, phk_stream_t s) {
  Prof prof_(FAM_ATTENTION, s, g ? 4.0 * (double)g->n_outer * g->n_inner * g->heads * g->n_q * g->n_k * g->dim_head : 0.0);
  PHK_REQUIRE(Qn && KVn && out && g, PHK_E_ARG, "phk_attention_small_bf16: null pointer");
  PHK_REQUIRE(g->n_outer > 0 && g->n_inner > 0 && g->heads > 0 && g->dim_head == 64 && g->n_q == g->n_k && g->n_q > 0 &&
                  g->n_q <= 16 && g->num_null_kv == 0, PHK_E_UNSUPPORTED,
              "phk_attention_small_bf16: needs dim_head 64, n_q == n_k <= 16 and no null-kv");
  PHK_REQUIRE(!g->causal || alibi_slopes, PHK_E_ARG, "phk_attention_small_bf16: causal attention takes ALiBi slopes");
  PHK_REQUIRE(g->q_tok % 2 == 0 && g->q_outer % 2 == 0 && g->q_inner % 2 == 0 && g->k_tok % 2 == 0 && g->k_outer % 2 == 0 &&
                  g->k_inner % 2 == 0 && g->o_tok % 2 == 0 && g->o_outer % 2 == 0 && g->o_inner % 2 == 0 &&
                  ((reinterpret_cast<uintptr_t>(Qn) | reinterpret_cast<uintptr_t>(KVn) | reinterpret_cast<uintptr_t>(out)) & 7) == 0,
              PHK_E_ARG, "phk_attention_small_bf16: operands must be 8-byte aligned with even strides");
  cudaStream_t st = to_stream(s);
  const int n = g->n_q;
#ifndef PHK_CUDA_EMU
  // warp-level tensor-core kernel: needs 16-byte aligned rows (token strides multiples of 8 elements)
  if (g->out_bf16 && g->q_tok % 8 == 0 && g->q_outer % 8 == 0 && g->q_inner % 8 == 0 && g->k_tok % 8 == 0 &&
      g->k_outer % 8 == 0 && g->k_inner % 8 == 0 && (g->heads * 64) % 8 == 0 &&
      ((reinterpret_cast<uintptr_t>(Qn) | reinterpret_cast<uintptr_t>(KVn)) & 15) == 0) {
    const int64_t npairs = (int64_t)g->n_outer * g->n_inner * g->heads;
    PHK_CUDA(launch_pdl(attention_small_mma_kernel, dim3((unsigned)((npairs + MMA_WARPS - 1) / MMA_WARPS)), dim3(MMA_WARPS * 32),
                        (size_t)0, st, (const __nv_bfloat16*)Qn, (const __nv_bfloat16*)KVn, alibi_slopes, (__nv_bfloat16*)out, *g));
    PHK_LAUNCH_CHECK();
    return 0;
  }
#endif
  if (n <= 3) return launch_attention_warp64<3, true>(Qn, KVn, nullptr, nullptr, alibi_slopes, out, *g, st);
  if (n <= 5) return launch_attention_warp64<5, true>(Qn, KVn, nullptr, nullptr, alibi_slopes, out, *g, st);
  if (n <= 9) return launch_attention_warp64<9, true>(Qn, KVn, nullptr, nullptr, alibi_slopes, out, *g, st);
  if (n <= 12) return launch_attention_warp64<12, true>(Qn, KVn, nullptr, nullptr, alibi_slopes, out, *g, st);
  return launch_attention_warp64<16, true>(Qn, KVn, nullptr, nullptr, alibi_slopes, out, *g, st);
}

#ifndef PHK_CUDA_EMU
// Packed cross-attention operands of every layer of a transformer call (see cross_kv_pack_kernel).  kv[l]: fp32 [ctx_b * L,
// 2 * heads * 64] (phk_maskgit_context_kv), null_kv[l]: [heads, 2 * nnull, 64], k_scale[l]: [64]; key_mask [ctx_b, L] or
// NULL.  pack: depth * ctx_b * heads * 8192 bytes, dead: depth * ctx_b * 32 floats.  nnull + L <= 32, depth <= 16.
extern "C" int phk_cross_kv_pack(const float* const* kv, const float* const* null_kv, const float* const* k_scale, int32_t depth,
                                 const uint8_t* key_mask, int32_t ctx_b, int32_t L, int32_t heads, int32_t nnull, void* pack,
                                 float* dead, phk_stream_t s) {
  PHK_REQUIRE(kv && null_kv && k_scale && pack && dead, PHK_E_ARG, "phk_cross_kv_pack: null pointer");
  PHK_REQUIRE(depth > 0 && depth <= 16 && ctx_b > 0 && L >= 0 && heads > 0 && nnull > 0 && nnull + L <= XK, PHK_E_UNSUPPORTED,
              "phk_cross_kv_pack: at most 16 layers and 32 key slots (null keys + text)");
  CrossPackArgs a;
  for (int l = 0; l < depth; ++l) {
    PHK_REQUIRE(kv[l] && null_kv[l] && k_scale[l], PHK_E_ARG, "phk_cross_kv_pack: null layer pointer");
    a.layer[l] = CrossPackLayer{kv[l], null_kv[l], k_scale[l]};
  }
  const int64_t warps = (int64_t)depth * ctx_b * heads * XK;
  PHK_CUDA(launch_pdl(cross_kv_pack_kernel, dim3((unsigned)((warps + 7) / 8)), dim3(256), (size_t)0, to_stream(s), a, key_mask,
                      (__nv_bfloat16*)pack, dead, (int)depth, (int)ctx_b, (int)L, (int)heads, (int)nnull));
  PHK_LAUNCH_CHECK();
  return 0;
}

// Cross-attention of one layer on the packed operands: Qn bf16 [n_seq * n_q, ld_q] (phk_gemm_bf16_qnorm), pack / dead of THIS
// layer (pack + l * ctx_b * heads * 8192 bytes, dead + l * ctx_b * 32), out bf16 [n_seq * n_q, ld_o].  Sequence s uses the text
// s % ctx_b; sequences >= null_from (or none: -1) attend to the null keys only (the CFG null half).
extern "C" int phk_attention_cross_packed(const void* Qn, int64_t ld_q, const void* pack, const float* dead, void* out,
                                          int64_t ld_o, int32_t n_seq, int32_t n_q, int32_t heads, int32_t ctx_b, int32_t nnull,
                                          int32_t null_from, phk_stream_t s) {
  Prof prof_(FAM_ATTENTION, s, 4.0 * (double)n_seq * heads * n_q * XK * 64);
  PHK_REQUIRE(Qn && pack && dead && out, PHK_E_ARG, "phk_attention_cross_packed: null pointer");
  PHK_REQUIRE(n_seq > 0 && n_seq <= 65535 && n_q > 0 && heads > 0 && heads <= 65535 && ctx_b > 0 && nnull > 0 && nnull <= XK,
              PHK_E_ARG, "phk_attention_cross_packed: bad geometry");
  PHK_REQUIRE(ld_q >= heads * 64 && ld_o >= heads * 64 && ld_q % 2 == 0 && ld_o % 2 == 0 &&
                  ((reinterpret_cast<uintptr_t>(Qn) | reinterpret_cast<uintptr_t>(out)) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(pack) & 15) == 0,
              PHK_E_ARG, "phk_attention_cross_packed: misaligned operands");
  dim3 grid((unsigned)((n_q + 127) / 128), (unsigned)heads, (unsigned)n_seq);
  PHK_CUDA(launch_pdl(attention_cross_packed_kernel, grid, dim3(256), (size_t)0, to_stream(s), (const __nv_bfloat16*)Qn, ld_q,
                      (const __nv_bfloat16*)pack, dead, (__nv_bfloat16*)out, ld_o, (int)n_q, (int)heads, (int)ctx_b, (int)nnull,
                      (int)null_from));
  PHK_LAUNCH_CHECK();
  return 0;
}
#endif

#ifndef PHK_CUDA_EMU
// Self-attention core for 16 < n <= 64 tokens per sequence on the bf16 operands phk_gemm_bf16_qkv writes (same arguments as
// phk_attention_tc_bf16): Qn [n_seq*n, ld_q], KVn [n_seq*n, ld_kv] (keys | values), bias fp32 [heads, n, n] or NULL ->
// out bf16 [n_seq*n, heads*64].
extern "C" int phk_attention_mid_bf16(const void* Qn, int64_t ld_q, const void* KVn, int64_t ld_kv, const float* bias,
                                      void* out_bf16, int32_t n_seq, int32_t n, int32_t heads, phk_stream_t s) {
  Prof prof_(FAM_ATTENTION, s, 4.0 * (double)n_seq * heads * n * n * 64);
  PHK_REQUIRE(Qn && KVn && out_bf16, PHK_E_ARG, "phk_attention_mid_bf16: null pointer");
  PHK_REQUIRE(n_seq > 0 && n_seq <= 65535 && n > 0 && n <= MID_N && heads > 0, PHK_E_ARG,
              "phk_attention_mid_bf16: at most 64 tokens per sequence, 65535 sequences");
  const int64_t I = (int64_t)heads * 64;
  PHK_REQUIRE(ld_q >= I && ld_kv >= 2 * I && ld_q % 8 == 0 && ld_kv % 8 == 0 &&
                  ((reinterpret_cast<uintptr_t>(Qn) | reinterpret_cast<uintptr_t>(KVn)) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(out_bf16) & 3) == 0,
              PHK_E_ARG, "phk_attention_mid_bf16: operands must be 16-byte aligned with leading dimensions multiple of 8");
  PHK_CUDA(launch_pdl(attention_mid_mma_kernel, dim3((unsigned)heads, (unsigned)n_seq), dim3(128), (size_t)0, to_stream(s),
                      (const __nv_bfloat16*)Qn, ld_q, (const __nv_bfloat16*)KVn, ld_kv, bias, (__nv_bfloat16*)out_bf16, I, (int)n,
                      (int)heads));
  PHK_LAUNCH_CHECK();
  return 0;
}
#endif
