// Tensor-core cosine-sim attention for long sequences (MaskGit self-attention, attention.py:146-181 with the 3-D
// continuous position bias, n = T'H'W' = 576..1024 tokens, dim_head 64), sm_90a (wgmma).
//
//   operands           : bf16, TOKEN-major as the projections write them: Qn [rows, heads*64] (l2-normalised, * q_scale * 8),
//                        KVn [rows, 2*heads*64] (keys normalised * k_scale | values) -- produced directly by the q / k,v
//                        projection GEMM's epilogue (phk_gemm_bf16_qkv) or, for fp32 projections, by attention_prep_kernel.
//                        4-D tensor maps (d, head, token, sequence) pick one head's tile out of the token-major rows, so no
//                        head-major copy exists; V is consumed as an MN-major B operand (rows = keys), so no transposed
//                        copy either.
//   phk_attention_tc   : one CTA per (64-query tile, head, sequence); keys streamed in chunks of 64 through a two-deep ring.
//       warps 0..3  one warpgroup: S[64x64] = Q K^T (wgmma, both operands in shared memory) into registers, + bias,
//                   online max / sum (fp32, a row shared by the four lanes of a quad), P = exp(s - m) packed to bf16
//                   in registers and used directly as the A operand of O[64x64] += P V (wgmma, A from registers).
//       warp 4      TMA producer (SWIZZLE_128B; out-of-range rows zero-filled).
//   S and P never leave the registers; 40 KB shared memory per CTA -> several CTAs per SM overlap MMA and softmax.
#include "phk_common.cuh"
#include "phk_sm90.cuh"
#include <cstdlib>
#include <mutex>
#include <unordered_map>

namespace phk {
namespace {

constexpr int AQ = 64;    // queries per CTA (wgmma M)
constexpr int AKC = 64;   // keys per chunk (N of S, K extent of PV)
constexpr int ADH = 64;   // dim_head
constexpr int ATHREADS = 128 + 32;  // one MMA / softmax warpgroup + the TMA producer warp
constexpr int ASTAGES = 2;
constexpr int SQ_BYTES = AQ * ADH * 2, SK_BYTES = AKC * ADH * 2, SV_BYTES = ADH * AKC * 2;
constexpr int ATT_SMEM = SQ_BYTES + ASTAGES * (SK_BYTES + SV_BYTES) + 128 + 1024;

struct AttTcParams {
  const float* bias;        // [heads, n_q, n_k] fp32 or NULL
  __nv_bfloat16* out;       // [.., heads*64] bf16; token i of sequence s at (s*o_seq + i*o_tok) elements
  int n_q, n_k, heads;
  int64_t o_seq, o_tok;
};

__global__ void __launch_bounds__(ATHREADS) attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                                const __grid_constant__ CUtensorMap tmK,
                                                                const __grid_constant__ CUtensorMap tmV,
                                                                AttTcParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base, sK = sQ + SQ_BYTES, sV = sK + ASTAGES * SK_BYTES;
  const uint32_t bars = sV + ASTAGES * SV_BYTES;
  const uint32_t b_q = bars, b_full = bars + 8, b_empty = b_full + 8 * ASTAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AQ, h = blockIdx.y, seq = blockIdx.z;
  const int nch = (p.n_k + AKC - 1) / AKC;

  if (threadIdx.x == 0) {
    mbar_init(b_q, 1);
    for (int s = 0; s < ASTAGES; ++s) { mbar_init(b_full + 8 * s, 1); mbar_init(b_empty + 8 * s, 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x == 128) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmQ) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmK) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmV) : "memory");
  }
  __syncthreads();
  pdl_wait();  // prologue above overlapped the previous kernel

  if (warp == 4) {
    if (lane == 0) {
      mbar_expect_tx(b_q, SQ_BYTES);
      tma_load_4d(&tmQ, b_q, sQ, 0, h, q0, seq);
      for (int j = 0; j < nch; ++j) {
        const int s = j % ASTAGES;
        mbar_wait(b_empty + 8 * s, ((j / ASTAGES) & 1) ^ 1);
        mbar_expect_tx(b_full + 8 * s, SK_BYTES + SV_BYTES);
        tma_load_4d(&tmK, b_full + 8 * s, sK + s * SK_BYTES, 0, h, j * AKC, seq);
        tma_load_4d(&tmV, b_full + 8 * s, sV + s * SV_BYTES, 0, h, j * AKC, seq);  // [64 keys][64 d]: MN-major B of P.V
      }
    }
    return;
  }
  // ---- MMA / softmax warpgroup: lane l of warp w holds rows 16w + l/4 (index 0) and + 8 (index 1) of the tile and
  // columns 8j + 2(l%4) + {0, 1}, j = 0..7, of S and O (wgmma accumulator fragment)
  const int t4 = lane & 3;
  const int rows[2] = {q0 + 16 * warp + (lane >> 2), q0 + 16 * warp + (lane >> 2) + 8};
  const float* brow[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) brow[i] = (p.bias && rows[i] < p.n_q) ? p.bias + ((int64_t)h * p.n_q + rows[i]) * p.n_k : nullptr;
  const bool bias_vec = (p.n_k % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.bias) & 7) == 0);
  constexpr float LOG2E = 1.4426950408889634f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  mbar_wait(b_q, 0);
  const uint64_t dq = gmma_desc(sQ);
  for (int j = 0; j < nch; ++j) {
    const int s = j % ASTAGES;
    mbar_wait(b_full + 8 * s, (j / ASTAGES) & 1);
    float sc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) sc[i] = 0.f;
    const uint64_t dk = gmma_desc(sK + s * SK_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < ADH / 16; ++k) wgmma_m64n64k16_ss<0>(sc, dq + 2 * k, dk + 2 * k, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    // + bias, padding keys -> -inf, chunk maximum per row
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int key = j * AKC + 8 * jj + 2 * t4;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float& a = sc[4 * jj + 2 * i];
        float& b = sc[4 * jj + 2 * i + 1];
        if (brow[i]) {
          if (bias_vec && key + 1 < p.n_k) {
            const float2 t = __ldg(reinterpret_cast<const float2*>(brow[i] + key));
            a += t.x; b += t.y;
          } else {
            if (key < p.n_k) a += __ldg(brow[i] + key);
            if (key + 1 < p.n_k) b += __ldg(brow[i] + key + 1);
          }
        }
        if (key >= p.n_k) a = -INFINITY;  // zero-filled padding keys
        if (key + 1 >= p.n_k) b = -INFINITY;
        mx[i] = fmaxf(mx[i], fmaxf(a, b));
      }
    }
    float alpha[2], m2[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
      const float m_new = fmaxf(m_run[i], mx[i]);  // finite: every chunk starts with a valid key
      alpha[i] = fast_ex2((m_run[i] - m_new) * LOG2E);  // 0 on the first chunk (m_run = -inf)
      m2[i] = m_new * LOG2E;
      m_run[i] = m_new;
    }
    // P = exp(s - m) -> bf16 A fragments of the P.V product (four K = 16 steps of 16 keys)
    uint32_t pa[4][4];
    float lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float p0 = fast_ex2(fmaf(sc[4 * jj + 2 * i], LOG2E, -m2[i]));
        const float p1 = fast_ex2(fmaf(sc[4 * jj + 2 * i + 1], LOG2E, -m2[i]));
        lsum[i] += p0 + p1;
        pa[jj >> 1][(jj & 1) * 2 + i] = pack_bf16x2(p0, p1);
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) l_run[i] = l_run[i] * alpha[i] + lsum[i];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      o[4 * jj] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
      o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
    }
    const uint64_t dv = gmma_desc_mn(sV + s * SV_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AKC / 16; ++k)  // 16 keys = two 8-row atoms of V = 2048 B (128 descriptor units) per step
      wgmma_m64n64k16_rs<1>(o, pa[k], dv + 128 * k, 1u);
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(b_empty + 8 * s);  // this warp is done with K and V of the slot
  }
  // row sums over the quad, normalise, bf16 out
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 1);
    l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 2);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (rows[i] >= p.n_q) continue;
    const float inv = 1.f / l_run[i];
    __nv_bfloat16* orow = p.out + (int64_t)seq * p.o_seq + (int64_t)rows[i] * p.o_tok + h * ADH;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
      *reinterpret_cast<uint32_t*>(orow + 8 * jj + 2 * t4) = pack_bf16x2(o[4 * jj + 2 * i] * inv, o[4 * jj + 2 * i + 1] * inv);
  }
}

// --------------------------------------------------------------------------------------------------------------
// prep (fp32 projection outputs only; the bf16 pipeline gets these operands from the GEMM epilogue): token-major fp32
// q [rows, I], kv [rows, 2I] -> token-major bf16 Qn [rows, I], KVn [rows, 2I]
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) attention_prep_kernel(const float* __restrict__ q, const float* __restrict__ kv,
                                                             const float* __restrict__ q_scale,
                                                             const float* __restrict__ k_scale,
                                                             __nv_bfloat16* __restrict__ Qn, __nv_bfloat16* __restrict__ KVn,
                                                             int64_t rows, int heads, float scale) {
  pdl_prologue();
  const int I = heads * 64;
  const int lane = threadIdx.x & 31;
  // lane owns dims (2 lane, 2 lane + 1) of one head: one 8-byte load per operand, one bf16x2 store per output
  const float2 qs = reinterpret_cast<const float2*>(q_scale)[lane], ks = reinterpret_cast<const float2*>(k_scale)[lane];
  const int64_t pairs = rows * heads;
  for (int64_t pr = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pr < pairs;
       pr += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const int64_t row = pr / heads;
    const int h = (int)(pr - row * heads);
    const float2 xq = reinterpret_cast<const float2*>(q + row * I + h * 64)[lane];
    const float2 xk = reinterpret_cast<const float2*>(kv + row * 2 * I + h * 64)[lane];
    const float2 xv = reinterpret_cast<const float2*>(kv + row * 2 * I + I + h * 64)[lane];
    // 1 / max(||x||, 1e-12) (F.normalize, attention.py:153-154); the fixed scale 8 (:157) is folded into q
    const float iq = 1.0f / fmaxf(sqrtf(warp_sum(xq.x * xq.x + xq.y * xq.y)), 1e-12f);
    const float ik = 1.0f / fmaxf(sqrtf(warp_sum(xk.x * xk.x + xk.y * xk.y)), 1e-12f);
    reinterpret_cast<uint32_t*>(Qn + row * I + h * 64)[lane] = pack_bf16x2((xq.x * iq) * qs.x * scale, (xq.y * iq) * qs.y * scale);
    reinterpret_cast<uint32_t*>(KVn + row * 2 * I + h * 64)[lane] = pack_bf16x2((xk.x * ik) * ks.x, (xk.y * ik) * ks.y);
    reinterpret_cast<uint32_t*>(KVn + row * 2 * I + I + h * 64)[lane] = pack_bf16x2(xv.x, xv.y);
  }
}


// one head's [tokens, 64] tile out of a token-major bf16 matrix [n_seq * n rows, ld elements]: dims (d, head, token,
// sequence), box [64 d][1][box_tok tokens][1], SWIZZLE_128B; tokens >= n are zero-filled (never the next sequence's)
int make_map_4d(const void* ptr, int64_t n, int64_t heads, int64_t n_seq, int64_t ld, int box_tok, CUtensorMap* out) {
  EncodeTiledFn fn = encode_fn();
  PHK_REQUIRE(fn, PHK_E_UNSUPPORTED, "cuTensorMapEncodeTiled not available from the driver");
  // dimension order (d, head, token, sequence): byte strides 128 < 2 ld < 2 n ld grow with the dimension index
  const cuuint64_t gdim[4] = {64, (cuuint64_t)heads, (cuuint64_t)n, (cuuint64_t)n_seq};
  const cuuint64_t gstride[3] = {128, (cuuint64_t)ld * 2, (cuuint64_t)n * (cuuint64_t)ld * 2};
  const cuuint32_t box[4] = {64, 1, (cuuint32_t)box_tok, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PHK_REQUIRE(r == CUDA_SUCCESS, PHK_E_ARG, "cuTensorMapEncodeTiled rejected an attention operand");
  return 0;
}

}  // namespace
}  // namespace phk

using namespace phk;

extern "C" int64_t phk_attention_tc_scratch_bytes(int32_t n_seq, int32_t n, int32_t heads) {
  return (int64_t)n_seq * n * heads * 64 * 3 * 2 + 2 * 256;   // Qn [rows, I] + KVn [rows, 2I], bf16
}

// Core on bf16 operands as phk_gemm_bf16_qkv writes them: Qn [n_seq*n, ld_q] (normalised, scaled), KVn [n_seq*n, ld_kv]
// (normalised keys in columns [0, heads*64), values in [heads*64, 2*heads*64)); bias fp32 [heads, n, n] or NULL
// -> out bf16 [n_seq*n, heads*64].
extern "C" int phk_attention_tc_bf16(const void* Qn, int64_t ld_q, const void* KVn, int64_t ld_kv, const float* bias,
                                     void* out_bf16, int32_t n_seq, int32_t n, int32_t heads, phk_stream_t s) {
  Prof prof_(FAM_ATTENTION, s, 4.0 * (double)n_seq * heads * n * n * 64);
  PHK_REQUIRE(Qn && KVn && out_bf16, PHK_E_ARG, "phk_attention_tc_bf16: null pointer");
  PHK_REQUIRE(n_seq > 0 && n > 0 && heads > 0 && n_seq <= 65535 && heads <= 65535, PHK_E_ARG, "phk_attention_tc_bf16: bad size");
  const int64_t I = (int64_t)heads * 64;
  PHK_REQUIRE(ld_q >= I && ld_kv >= 2 * I && ld_q % 8 == 0 && ld_kv % 8 == 0 &&
                  ((reinterpret_cast<uintptr_t>(Qn) | reinterpret_cast<uintptr_t>(KVn) | reinterpret_cast<uintptr_t>(out_bf16)) & 15) == 0,
              PHK_E_ARG, "phk_attention_tc_bf16: operands must be 16-byte aligned with leading dimensions multiple of 8 (TMA)");
  cudaStream_t st = to_stream(s);
  CUtensorMap tq, tk, tv;
  PHK_TRY(make_map_4d(Qn, n, heads, n_seq, ld_q, AQ, &tq));
  PHK_TRY(make_map_4d(KVn, n, heads, n_seq, ld_kv, AKC, &tk));
  PHK_TRY(make_map_4d(reinterpret_cast<const __nv_bfloat16*>(KVn) + I, n, heads, n_seq, ld_kv, AKC, &tv));
  AttTcParams p{bias, (__nv_bfloat16*)out_bf16, n, n, heads, (int64_t)n * heads * 64, (int64_t)heads * 64};
  dim3 grid((unsigned)((n + AQ - 1) / AQ), (unsigned)heads, (unsigned)n_seq);
  PHK_CUDA(launch_pdl(attention_tc_kernel, dim3(grid), dim3(ATHREADS), (size_t)(ATT_SMEM), st, tq, tk, tv, p));
  PHK_LAUNCH_CHECK();
  return 0;
}

// Self-attention core on tensor cores from fp32 projections: q fp32 [n_seq*n, heads*64], kv fp32 [n_seq*n, 2*heads*64]
// (token-major), bias fp32 [heads, n, n] or NULL -> out bf16 [n_seq*n, heads*64].  dim_head 64, no null-kv, no key
// mask, not causal (everything else takes phk_attention).  scratch >= phk_attention_tc_scratch_bytes.
extern "C" int phk_attention_tc(const float* q, const float* kv, const float* q_scale, const float* k_scale,
                                const float* bias, void* out_bf16, int32_t n_seq, int32_t n, int32_t heads,
                                float scale, void* scratch, int64_t scratch_bytes, phk_stream_t s) {
  PHK_REQUIRE(q && kv && q_scale && k_scale && out_bf16 && scratch, PHK_E_ARG, "phk_attention_tc: null pointer");
  PHK_REQUIRE(n_seq > 0 && n > 0 && heads > 0 && n_seq <= 65535 && heads <= 65535, PHK_E_ARG, "phk_attention_tc: bad size");
  PHK_REQUIRE(scratch_bytes >= phk_attention_tc_scratch_bytes(n_seq, n, heads), PHK_E_WORKSPACE,
              "phk_attention_tc: scratch too small");
  cudaStream_t st = to_stream(s);
  const int64_t rows = (int64_t)n_seq * n, I = (int64_t)heads * 64;
  auto align = [](char* p) { return (char*)(((uintptr_t)p + 255) & ~(uintptr_t)255); };
  __nv_bfloat16* Qn = (__nv_bfloat16*)align((char*)scratch);
  __nv_bfloat16* KVn = (__nv_bfloat16*)align((char*)Qn + rows * I * 2);
  {
    Prof prof_(FAM_ATTENTION, s, 0.0);
    const int64_t pairs = rows * heads;
    const unsigned blocks = (unsigned)((pairs + 7) / 8 < kNumSMs * 16 ? (pairs + 7) / 8 : kNumSMs * 16);
    PHK_CUDA(launch_pdl(attention_prep_kernel, dim3(blocks), dim3(256), (size_t)(0), st, q, kv, q_scale, k_scale, Qn, KVn, rows,
                        (int)heads, scale));
    PHK_LAUNCH_CHECK();
  }
  return phk_attention_tc_bf16(Qn, I, KVn, 2 * I, bias, out_bf16, n_seq, n, heads, s);
}
