// Cosine-similarity VectorQuantize lookup (the reference's non-LFQ tokenizer, `lookup_free_quantization=False`:
// cvivit.py:321 VectorQuantize(dim, codebook_size, use_cosine_sim=True); forward :568-570, restated in oracle/lfq.py):
//     ids[r] = argmax_c  l2norm(x[r]) . embed[c]
// The codebook rows are unit vectors and the positive factor 1/|x[r]| does not move an argmax, so the ids are the
// arg-max rows of the product x . embed^T -- (tokens x K x dim), 309 GFLOP at BASELINE configs[1], more than the encoder.
//   fp32 (parity):  phk_gemm_f32 into a [rows, K] strip of the caller's scratch + argmax_rows_kernel (first maximum wins,
//                   like torch.argmax), strip by strip so the similarities never need more than the scratch holds;
//   bf16:           the fused wgmma head (phk_head_sample at temperature 0 = pure argmax, phenaki_pytorch.py:493): the
//                   [tokens, K] similarities never leave the SM.
#include "phk_common.cuh"

namespace phk {
namespace {

// one CTA per row: arg-max over K columns, lowest index on ties
__global__ void __launch_bounds__(256) argmax_rows_kernel(const float* __restrict__ x, int64_t ld, int K,
                                                          int64_t* __restrict__ ids) {
  pdl_prologue();
  __shared__ float s_v[8];
  __shared__ int s_i[8];
  const float* row = x + (int64_t)blockIdx.x * ld;
  float best = -FLT_MAX;
  int bi = 0x7fffffff;
  for (int c = threadIdx.x; c < K; c += blockDim.x) {
    const float v = row[c];
    if (v > best || (v == best && c < bi)) { best = v; bi = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { s_v[w] = best; s_i[w] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k)
      if (s_v[k] > best || (s_v[k] == best && s_i[k] < bi)) { best = s_v[k]; bi = s_i[k]; }
    ids[blockIdx.x] = bi;
  }
}

int64_t a256(int64_t v) { return (v + 255) & ~int64_t(255); }

}  // namespace
}  // namespace phk

using namespace phk;

extern "C" int64_t phk_vq_cosine_scratch_bytes(int64_t rows, int32_t K, int32_t prec) {
  if (rows <= 0 || K <= 0) return -1;
  if (prec == PHK_PREC_BF16) return a256(rows) + a256(rows * 8) + a256(phk_head_sample_scratch_bytes((int32_t)rows)) + 512;
  const int64_t strip = rows < 1024 ? rows : 1024;  // similarities of at most 1024 tokens at a time
  return a256(strip * (int64_t)K * 4) + 512;
}

extern "C" int phk_vq_cosine_ids(const void* x, const float* codebook, const void* codebook_h, int64_t* ids, int64_t rows,
                                 int32_t dim, int32_t K, void* scratch, int64_t scratch_bytes, int32_t prec,
                                 phk_stream_t s) {
  PHK_REQUIRE(x && ids && scratch, PHK_E_ARG, "phk_vq_cosine_ids: null pointer");
  PHK_REQUIRE(rows > 0 && dim > 0 && K > 0, PHK_E_ARG, "phk_vq_cosine_ids: bad size");
  PHK_REQUIRE(scratch_bytes >= phk_vq_cosine_scratch_bytes(rows, K, prec), PHK_E_WORKSPACE, "phk_vq_cosine_ids: scratch too small");
  char* base = (char*)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
  cudaStream_t st = to_stream(s);
  if (prec == PHK_PREC_BF16) {  // x bf16 [rows, dim]
    PHK_REQUIRE(codebook_h && dim % 8 == 0 && dim <= 512, PHK_E_UNSUPPORTED,
                "phk_vq_cosine_ids: bf16 mode needs the bf16 codebook, dim % 8 == 0 and dim <= 512");
    uint8_t* ones = (uint8_t*)base;
    int64_t* dummy = (int64_t*)(base + a256(rows));
    char* hs = base + a256(rows) + a256(rows * 8);
    PHK_CUDA(cudaMemsetAsync(ones, 1, rows, st));
    // temperature 0: the head's gumbel term is negligible against logit / 1e-10 -> the arg-max of the similarities
    return phk_head_sample(x, dim, rows, codebook_h, dim, nullptr, (int32_t)rows, K, dim, 0.0f, 0, 0, ones, dummy, ids,
                           nullptr, hs, phk_head_sample_scratch_bytes((int32_t)rows), s);
  }
  PHK_REQUIRE(prec == PHK_PREC_F32 && codebook, PHK_E_ARG, "phk_vq_cosine_ids: fp32 mode needs the fp32 codebook");
  float* sim = (float*)base;
  const int64_t strip = rows < 1024 ? rows : 1024;
  const float* xf = (const float*)x;
  for (int64_t r0 = 0; r0 < rows; r0 += strip) {
    const int64_t nr = rows - r0 < strip ? rows - r0 : strip;
    PHK_TRY(phk_gemm_f32(xf + r0 * dim, dim, codebook, dim, sim, K, nr, K, dim, nullptr, nullptr, 0, 0, 0, s));
    PHK_CUDA(launch_pdl(argmax_rows_kernel, dim3((unsigned)nr), dim3(256), (size_t)0, st, (const float*)sim, (int64_t)K, K, ids + r0));
    PHK_LAUNCH_CHECK();
  }
  return 0;
}
