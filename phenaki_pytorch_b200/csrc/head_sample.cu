// Fused logits head of the sampling loop (sm_90a): logits GEMM + bias + gumbel noise + argmax + online softmax,
// reduced over the vocabulary inside the kernel -- the (b, n, V) logits never exist in memory
// (phenaki_pytorch.py:213 to_logits, :161 classifier-free guidance, :83-93 gumbel_sample, :506-509, :547-550).
//
// Classifier-free guidance is folded BEFORE the head: to_logits is linear, so
//     null + (cond - null) * s  ==  to_logits(e_null + s * (e_cond - e_null))
// and the guided embedding e_cfg (one row per token, produced by phk_layernorm_cfg from the two final-norm rows) is the
// only A operand: half the FLOPs of the reference's two logits GEMMs and no cond/null pairing in the epilogue.
//
// One CTA owns 128 tokens and a contiguous slice of the vocabulary:
//   warpgroup 0     TMA (one thread): the 128 x dim A panel is loaded ONCE and stays resident in shared memory
//                   (dim <= 512: 128 KB); W tiles (128 vocabulary rows x 64) stream through a 4-stage ring -> L2 traffic
//                   is W only.
//   warpgroups 1..4 each multiplies one 64-token x 64-column quadrant of the 128 x 128 logits tile (wgmma) and works on
//                   its accumulator fragment in registers: Philox4x32-7 noise (phk_common.cuh; counter layout and gumbel
//                   transform of phk_sample_tokens), running (argmax of l/T + g, l at argmax, max l, sum exp) per row.
// Partials per (token, vocabulary slice) are merged by head_finalize_kernel (pred, 1 - softmax(l)[pred], mask).
#include "phk_common.cuh"
#include "phk_sm90.cuh"
#include <mutex>

namespace phk {
namespace {

constexpr int HM = 128, HN = 128, HK = 64, HSTAGES = 4;
constexpr int H_MATH_WARPS = 16;
constexpr int HTHREADS = 128 + H_MATH_WARPS * 32;  // 640
constexpr int HSTAGE_BYTES = HN * HK * 2;          // 16 KB
constexpr int H_MAX_KB = 8;                        // dim <= 512
constexpr int H_EX_BYTES = HM * 6 * 4;             // exchange buffer of the merge of the two column halves
constexpr int H_SMEM = H_MAX_KB * HM * HK * 2 + HSTAGES * HSTAGE_BYTES + 256 + H_EX_BYTES + 1024;

struct HeadParams {
  const float* bias;
  int n_tokens, V, K, n_tiles, n_splits, tiles_per_split;
  float inv_T;
  unsigned long long seed, offset;
  const unsigned long long* rng;  // optional device {seed, offset} overriding the two above (see phk_head_sample_rng)
  float4* part_f;  // [n_tokens, n_splits] {best_y, l_at_best, max_l, sum_exp}
  int* part_i;     // [n_tokens, n_splits] argmax index
};

struct HeadRun {
  float best, lbest, mx, ssum;
  int bidx;
};
// merge of two partial states of one token: the larger perturbed logit (the smaller index on ties), log-sum-exp sums
__device__ __forceinline__ void head_merge(HeadRun& a, float oy, float ol, float om, float os, int oi) {
  if (oy > a.best || (oy == a.best && oi < a.bidx)) { a.best = oy; a.bidx = oi; a.lbest = ol; }
  const float nm = fmaxf(a.mx, om);
  a.ssum = a.ssum * __expf(a.mx - nm) + os * __expf(om - nm);
  a.mx = nm;
}

__global__ void __launch_bounds__(HTHREADS, 1) head_sample_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                  const __grid_constant__ CUtensorMap tmB,
                                                                  HeadParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const int num_kb = (p.K + HK - 1) / HK;
  const uint32_t sA = base;                                   // num_kb x [128 x 64] resident A panel
  const uint32_t sB = base + H_MAX_KB * HM * HK * 2;          // ring
  const uint32_t bars = sB + HSTAGES * HSTAGE_BYTES;
  const uint32_t bar_afull = bars, bar_full = bars + 8, bar_empty = bar_full + 8 * HSTAGES;
  float* ex = reinterpret_cast<float*>(base_ptr + H_MAX_KB * HM * HK * 2 + HSTAGES * HSTAGE_BYTES + 256);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tile = blockIdx.x / p.n_splits, split = blockIdx.x % p.n_splits;
  const int n_begin = split * p.tiles_per_split;
  const int my_tiles = max(0, min(p.tiles_per_split, p.n_tiles - n_begin));

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    mbar_init(bar_afull, 1);
    for (int s = 0; s < HSTAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, H_MATH_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();

  if (warp < 4) {
    if (warp == 0 && lane == 0 && my_tiles > 0) {
      mbar_expect_tx(bar_afull, (uint32_t)num_kb * HM * HK * 2);
      for (int kb = 0; kb < num_kb; ++kb) tma_load_2d(&tmA, bar_afull, sA + kb * HM * HK * 2, kb * HK, m_tile * HM);
      int stage = 0;
      uint32_t phase = 0;
      for (int it = 0; it < my_tiles; ++it) {
        const int n0 = (n_begin + it) * HN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bar_empty + 8 * stage, phase ^ 1);
          mbar_expect_tx(bar_full + 8 * stage, HSTAGE_BYTES);
          tma_load_2d(&tmB, bar_full + 8 * stage, sB + stage * HSTAGE_BYTES, kb * HK, n0);
          if (++stage == HSTAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== MMA + math warps =====================
    const int mw = warp - 4;
    const int wg = mw >> 2, w = mw & 3;
    const int rq = (wg & 1) * 64, cq = (wg >> 1) * 64;  // this warpgroup's quadrant of the tile
    const int t4 = lane & 3;
    int tl[2], tok[2];
    unsigned long long ctr0[2];
    // noise key: by value, or read from device memory so that a captured CUDA graph draws fresh noise on every replay
    const unsigned long long seed = p.rng ? p.rng[0] : p.seed;
    const unsigned long long off = p.rng ? p.rng[1] : p.offset;
    HeadRun run[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      tl[i] = rq + 16 * w + (lane >> 2) + 8 * i;
      tok[i] = m_tile * HM + tl[i];
      ctr0[i] = off + (unsigned long long)tok[i] * (unsigned long long)((p.V + 3) / 4);
      run[i] = HeadRun{-FLT_MAX, 0.f, -FLT_MAX, 0.f, 0x7fffffff};
    }
    constexpr float LOG2E = 1.4426950408889634f;
    if (my_tiles > 0) mbar_wait(bar_afull, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0; it < my_tiles; ++it) {
      float d[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) d[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase);
        const uint64_t da = gmma_desc(sA + kb * HM * HK * 2 + rq * 128);
        const uint64_t db = gmma_desc(sB + stage * HSTAGE_BYTES + cq * 128);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < HK / 16; ++k) wgmma_m64n64k16_ss<0>(d, da + 2 * k, db + 2 * k, 1u);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * stage);
        if (++stage == HSTAGES) { stage = 0; phase ^= 1; }
      }
      // columns v, v + 1 (v even) of each row, in increasing v: Philox block v / 4 supplies draws v % 4 and v % 4 + 1
      // (the same (token, v) -> noise map as phk_sample_tokens)
      const int v_tile = (n_begin + it) * HN + cq + 2 * t4;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int v = v_tile + 8 * jj;
        if (v >= p.V) break;
        const bool in1 = v + 1 < p.V;
        float bb[2] = {0.f, 0.f};
        if (p.bias) { bb[0] = __ldg(p.bias + v); if (in1) bb[1] = __ldg(p.bias + v + 1); }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          if (tok[i] >= p.n_tokens) continue;
          uint32_t rnd[4];
          const unsigned long long ctr = ctr0[i] + (unsigned long long)(v >> 2);
          philox4x32<kNoiseRounds>((uint32_t)ctr, (uint32_t)(ctr >> 32), 0u, 0u, (uint32_t)seed, (uint32_t)(seed >> 32), rnd);
          const uint32_t r0 = (v & 2) ? rnd[2] : rnd[0], r1 = (v & 2) ? rnd[3] : rnd[1];
          const float l0 = d[4 * jj + 2 * i] + bb[0];
          const float l1 = in1 ? d[4 * jj + 2 * i + 1] + bb[1] : -FLT_MAX;
          HeadRun& a = run[i];
          const float y0 = fmaf(l0, p.inv_T, gumbel_from_bits(r0));
          if (y0 > a.best) { a.best = y0; a.bidx = v; a.lbest = l0; }
          if (in1) {
            const float y1 = fmaf(l1, p.inv_T, gumbel_from_bits(r1));
            if (y1 > a.best) { a.best = y1; a.bidx = v + 1; a.lbest = l1; }
          }
          const float gm = fmaxf(l0, l1);
          if (gm > a.mx) { a.ssum *= fast_ex2((a.mx - gm) * LOG2E); a.mx = gm; }
          const float mxs = a.mx * LOG2E;
          a.ssum += fast_ex2(fmaf(l0, LOG2E, -mxs));
          if (in1) a.ssum += fast_ex2(fmaf(l1, LOG2E, -mxs));
        }
      }
    }
    // merge the four lanes of a quad (same rows), then the two column halves of every token
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        const float oy = __shfl_xor_sync(0xffffffffu, run[i].best, o), ol = __shfl_xor_sync(0xffffffffu, run[i].lbest, o);
        const float om = __shfl_xor_sync(0xffffffffu, run[i].mx, o), os = __shfl_xor_sync(0xffffffffu, run[i].ssum, o);
        const int oi = __shfl_xor_sync(0xffffffffu, run[i].bidx, o);
        head_merge(run[i], oy, ol, om, os, oi);
      }
      if (cq == 64 && t4 == 0) {
        float* e = ex + tl[i] * 6;
        e[0] = run[i].best; e[1] = run[i].lbest; e[2] = run[i].mx; e[3] = run[i].ssum; e[4] = __int_as_float(run[i].bidx);
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(H_MATH_WARPS * 32) : "memory");
    if (cq == 0 && t4 == 0) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (tok[i] >= p.n_tokens) continue;
        const float* e = ex + tl[i] * 6;
        head_merge(run[i], e[0], e[1], e[2], e[3], __float_as_int(e[4]));
        const int64_t slot = (int64_t)tok[i] * p.n_splits + split;
        p.part_f[slot] = make_float4(run[i].best, run[i].lbest, run[i].mx, run[i].ssum);
        p.part_i[slot] = run[i].bidx;
      }
    }
  }
}

// combines the per-slice partials: pred = argmax, score = 1 - softmax(l)[pred] (phenaki_pytorch.py:506-509, 547-550);
// same output semantics as sample_tokens_kernel
__global__ void head_finalize_kernel(const float4* __restrict__ part_f, const int* __restrict__ part_i, int n_splits,
                                     int n_tokens, const uint8_t* __restrict__ mask, int64_t* __restrict__ ids,
                                     int64_t* __restrict__ pred_out, float* __restrict__ score_out) {
  pdl_prologue();
  const int tok = blockIdx.x * blockDim.x + threadIdx.x;
  if (tok >= n_tokens) return;
  float by = -FLT_MAX, bl = 0.f, m = -FLT_MAX, ssum = 0.f;
  int bi = 0x7fffffff;
  for (int s = 0; s < n_splits; ++s) {
    const float4 f = part_f[(int64_t)tok * n_splits + s];
    const int i = part_i[(int64_t)tok * n_splits + s];
    if (f.x > by || (f.x == by && i < bi)) { by = f.x; bi = i; bl = f.y; }
    const float nm = fmaxf(m, f.z);
    ssum = ssum * __expf(m - nm) + f.w * __expf(f.z - nm);
    m = nm;
  }
  const float prob = __expf(bl - m) / ssum;
  const bool mk = mask ? mask[tok] != 0 : true;
  if (pred_out) pred_out[tok] = bi;
  if (ids && mk) ids[tok] = bi;
  if (score_out) score_out[tok] = mk ? 1.0f - prob : -1e4f;
}

// e_cfg = LN(x_null) + s * (LN(x_cond) - LN(x_null)) -> bf16; warp per token, dim % 128 == 0, dim <= 1024.
// The final norm_out of the transformer (attention.py:308,332) for both halves of a CFG pair, combined with the
// guidance scale BEFORE the (linear) logits head.
template <int VEC>
__global__ void __launch_bounds__(256) ln_cfg_kernel(const float* __restrict__ xc, const float* __restrict__ xn,
                                                     const float* __restrict__ g, const float* __restrict__ b,
                                                     float scale, __nv_bfloat16* __restrict__ out, int64_t rows, int dim) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  float4 o[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) o[j] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const float4* xr = reinterpret_cast<const float4*>((pass ? xn : xc) + row * dim);
    float4 v[VEC];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < VEC; ++j) { v[j] = xr[lane + 32 * j]; s += (v[j].x + v[j].y) + (v[j].z + v[j].w); }
    const float mean = warp_sum(s) / (float)dim;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float a = v[j].x - mean, bb = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
      q += (a * a + bb * bb) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)dim + 1e-5f);
    const float w = pass ? (1.0f - scale) : scale;  // null + s*(cond - null) = s*cond + (1-s)*null
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float4 gg = reinterpret_cast<const float4*>(g)[lane + 32 * j], bb = reinterpret_cast<const float4*>(b)[lane + 32 * j];
      o[j].x += w * ((v[j].x - mean) * rstd * gg.x + bb.x);
      o[j].y += w * ((v[j].y - mean) * rstd * gg.y + bb.y);
      o[j].z += w * ((v[j].z - mean) * rstd * gg.z + bb.z);
      o[j].w += w * ((v[j].w - mean) * rstd * gg.w + bb.w);
    }
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j)
    reinterpret_cast<uint2*>(out + row * dim)[lane + 32 * j] = make_uint2(pack_bf16x2(o[j].x, o[j].y), pack_bf16x2(o[j].z, o[j].w));
}

int make_map_2d(const void* ptr, int64_t rows, int64_t cols, int64_t ld, CUtensorMap* out) {
  EncodeTiledFn fn = encode_fn();
  PHK_REQUIRE(fn, PHK_E_UNSUPPORTED, "cuTensorMapEncodeTiled not available from the driver");
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)HK, 128};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PHK_REQUIRE(r == CUDA_SUCCESS, PHK_E_ARG, "cuTensorMapEncodeTiled rejected a head operand (alignment / pitch)");
  return 0;
}

}  // namespace
}  // namespace phk

using namespace phk;

extern "C" int phk_layernorm_cfg(const float* x_cond, const float* x_null, const float* gamma, const float* beta,
                                 float cond_scale, void* out_bf16, int64_t rows, int32_t dim, phk_stream_t s) {
  Prof prof_(FAM_LAYERNORM, s, (double)rows * dim * 10.0);
  PHK_REQUIRE(x_cond && x_null && gamma && beta && out_bf16, PHK_E_ARG, "phk_layernorm_cfg: null pointer");
  PHK_REQUIRE(rows >= 0 && dim > 0 && dim % 128 == 0 && dim <= 1024, PHK_E_UNSUPPORTED,
              "phk_layernorm_cfg: dim must be a multiple of 128, <= 1024");
  if (rows == 0) return 0;
  cudaStream_t st = to_stream(s);
  const dim3 grid((unsigned)((rows + 7) / 8)), block(256);
  __nv_bfloat16* o = (__nv_bfloat16*)out_bf16;
  switch (dim / 128) {
    case 1: PHK_CUDA(launch_pdl(ln_cfg_kernel<1>, grid, block, 0, st, x_cond, x_null, gamma, beta, cond_scale, o, rows, dim)); break;
    case 2: PHK_CUDA(launch_pdl(ln_cfg_kernel<2>, grid, block, 0, st, x_cond, x_null, gamma, beta, cond_scale, o, rows, dim)); break;
    case 3: PHK_CUDA(launch_pdl(ln_cfg_kernel<3>, grid, block, 0, st, x_cond, x_null, gamma, beta, cond_scale, o, rows, dim)); break;
    case 4: PHK_CUDA(launch_pdl(ln_cfg_kernel<4>, grid, block, 0, st, x_cond, x_null, gamma, beta, cond_scale, o, rows, dim)); break;
    case 5: PHK_CUDA(launch_pdl(ln_cfg_kernel<5>, grid, block, 0, st, x_cond, x_null, gamma, beta, cond_scale, o, rows, dim)); break;
    case 6: PHK_CUDA(launch_pdl(ln_cfg_kernel<6>, grid, block, 0, st, x_cond, x_null, gamma, beta, cond_scale, o, rows, dim)); break;
    case 7: PHK_CUDA(launch_pdl(ln_cfg_kernel<7>, grid, block, 0, st, x_cond, x_null, gamma, beta, cond_scale, o, rows, dim)); break;
    default: PHK_CUDA(launch_pdl(ln_cfg_kernel<8>, grid, block, 0, st, x_cond, x_null, gamma, beta, cond_scale, o, rows, dim)); break;
  }
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t phk_head_sample_scratch_bytes(int32_t n_tokens) {
  const int m_tiles = (n_tokens + HM - 1) / HM;
  const int n_splits = m_tiles >= kNumSMs ? 1 : kNumSMs / m_tiles;
  return (int64_t)n_tokens * n_splits * 20 + 512;
}

extern "C" int phk_head_sample(const void* emb, int64_t ld_emb, int64_t emb_rows, const void* W, int64_t ldw,
                               const float* bias, int32_t n_tokens, int32_t V, int32_t dim, float temperature,
                               uint64_t seed, uint64_t offset, const uint8_t* mask, int64_t* ids, int64_t* pred_out,
                               float* score_out, void* scratch, int64_t scratch_bytes, phk_stream_t s) {
  return phk_head_sample_rng(emb, ld_emb, emb_rows, W, ldw, bias, n_tokens, V, dim, temperature, seed, offset, nullptr, mask,
                             ids, pred_out, score_out, scratch, scratch_bytes, s);
}

extern "C" int phk_head_sample_rng(const void* emb, int64_t ld_emb, int64_t emb_rows, const void* W, int64_t ldw,
                                   const float* bias, int32_t n_tokens, int32_t V, int32_t dim, float temperature,
                                   uint64_t seed, uint64_t offset, const uint64_t* rng_state, const uint8_t* mask,
                                   int64_t* ids, int64_t* pred_out, float* score_out, void* scratch, int64_t scratch_bytes,
                                   phk_stream_t s) {
  Prof prof_(FAM_GEMM_BF16, s, 2.0 * (double)n_tokens * V * dim);
  PHK_REQUIRE(emb && W && scratch, PHK_E_ARG, "phk_head_sample: null pointer");
  PHK_REQUIRE(n_tokens > 0 && V > 0 && dim > 0 && ld_emb >= dim && ldw >= dim && emb_rows >= n_tokens, PHK_E_ARG,
              "phk_head_sample: bad size");
  PHK_REQUIRE(dim <= H_MAX_KB * HK, PHK_E_UNSUPPORTED, "phk_head_sample: dim > 512 (A panel must fit in shared memory)");
  PHK_REQUIRE(ld_emb % 8 == 0 && ldw % 8 == 0 && (reinterpret_cast<uintptr_t>(emb) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(W) & 15) == 0,
              PHK_E_ARG, "phk_head_sample: operands must be 16-byte aligned with leading dimensions multiple of 8 (TMA)");
  PHK_REQUIRE(scratch_bytes >= phk_head_sample_scratch_bytes(n_tokens), PHK_E_WORKSPACE, "phk_head_sample: scratch too small");
  const int m_tiles = (n_tokens + HM - 1) / HM;
  const int n_tiles = (V + HN - 1) / HN;
  int n_splits = m_tiles >= kNumSMs ? 1 : kNumSMs / m_tiles;
  if (n_splits > n_tiles) n_splits = n_tiles;
  const int tps = (n_tiles + n_splits - 1) / n_splits;
  n_splits = (n_tiles + tps - 1) / tps;  // no empty vocabulary splits (e.g. 512 tiles over 49 splits of 11: 47 are enough)
  CUtensorMap ta, tb;
  PHK_TRY(make_map_2d(emb, emb_rows, dim, ld_emb, &ta));  // rows beyond emb_rows are zero-filled by the TMA unit
  PHK_TRY(make_map_2d(W, V, dim, ldw, &tb));
  char* sc = (char*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
  float4* part_f = (float4*)sc;
  int* part_i = (int*)(sc + (int64_t)n_tokens * n_splits * 16);
  const float T = temperature > 1e-10f ? temperature : 1e-10f;
  HeadParams p{bias, n_tokens, V, dim, n_tiles, n_splits, tps, 1.0f / T, (unsigned long long)seed,
               (unsigned long long)offset, reinterpret_cast<const unsigned long long*>(rng_state), part_f, part_i};
  cudaStream_t st = to_stream(s);
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(head_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, H_SMEM));
    mark_configured(&configured_mask);
  }
  PHK_CUDA(launch_pdl(head_sample_kernel, dim3(m_tiles * n_splits), dim3(HTHREADS), (size_t)H_SMEM, st, ta, tb, p));
  PHK_LAUNCH_CHECK();
  PHK_CUDA(launch_pdl(head_finalize_kernel, dim3((n_tokens + 127) / 128), dim3(128), (size_t)0, st, part_f, part_i,
                      n_splits, n_tokens, mask, ids, pred_out, score_out));
  PHK_LAUNCH_CHECK();
  return 0;
}
