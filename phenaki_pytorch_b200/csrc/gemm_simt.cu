// fp32 FFMA GEMM for the parity mode: C[map(m), n] = sum_k A[m,k] * W[n,k] (+bias) (+residual).
// nn.Linear semantics (attention.py:49-52, 120-126; cvivit.py:276, 283).  fp32 operands and
// fp32 accumulation keep the C-ViViT token ids identical to the fp32 reference (SURVEY H1);
// the tensor-core path lives in gemm_wgmma.cu.
//
// 128x128x16 CTA tile, 256 threads, 8x8 register micro-tile, double-buffered shared memory
// (k-major so the inner loop reads two float4 per operand with no bank conflicts).
#include "phk_common.cuh"

namespace phk {

constexpr int BM = 128, BN = 128, BK = 16, THREADS = 256;

struct RowMap {
  int64_t seg_len, seg_stride, seg_off;
  __device__ __forceinline__ int64_t operator()(int64_t m) const {
    if (seg_len <= 0) return m;
    const int64_t q = m / seg_len;
    return q * seg_stride + seg_off + (m - q * seg_len);
  }
};

// loads a (rows x BK) slab of a K-contiguous matrix into registers: each thread 2 x float4
template <bool ALIGNED>
__device__ __forceinline__ void load_slab(const float* __restrict__ P, int64_t ld, int64_t row0, int64_t nrows,
                                          int k0, int K, float4 (&r)[2]) {
  // 128 rows x 16 k = 512 float4; thread t handles float4 index t and t+256
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int f = threadIdx.x + i * THREADS;
    const int row = f >> 2;       // 4 float4 per row
    const int kq = (f & 3) << 2;  // k offset within the slab
    const int64_t gr = row0 + row;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gr < nrows) {
      const float* p = P + gr * ld + k0 + kq;
      if (ALIGNED && k0 + kq + 3 < K) {
        v = __ldg(reinterpret_cast<const float4*>(p));
      } else {
        if (k0 + kq + 0 < K) v.x = __ldg(p + 0);
        if (k0 + kq + 1 < K) v.y = __ldg(p + 1);
        if (k0 + kq + 2 < K) v.z = __ldg(p + 2);
        if (k0 + kq + 3 < K) v.w = __ldg(p + 3);
      }
    }
    r[i] = v;
  }
}

__device__ __forceinline__ void store_slab(float (*S)[BM + 4], const float4 (&r)[2]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int f = threadIdx.x + i * THREADS;
    const int row = f >> 2;
    const int kq = (f & 3) << 2;
    S[kq + 0][row] = r[i].x;
    S[kq + 1][row] = r[i].y;
    S[kq + 2][row] = r[i].z;
    S[kq + 3][row] = r[i].w;
  }
}

template <bool ALIGNED>
__global__ void __launch_bounds__(THREADS, 2) gemm_f32_kernel(const float* __restrict__ A, int64_t lda,
                                                              const float* __restrict__ W, int64_t ldw,
                                                              float* __restrict__ C, int64_t ldc, int64_t M, int N,
                                                              int K, const float* __restrict__ bias,
                                                              const float* __restrict__ residual, RowMap map) {
  pdl_prologue();
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];
  const int64_t m0 = (int64_t)blockIdx.y * BM;
  const int n0 = blockIdx.x * BN;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];
  load_slab<ALIGNED>(A, lda, m0, M, 0, K, ra);
  load_slab<ALIGNED>(W, ldw, n0, N, 0, K, rb);
  store_slab(As[0], ra);
  store_slab(Bs[0], rb);
  __syncthreads();
  const int nk = (K + BK - 1) / BK;
  for (int kt = 0; kt < nk; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nk) {
      load_slab<ALIGNED>(A, lda, m0, M, (kt + 1) * BK, K, ra);
      load_slab<ALIGNED>(W, ldw, n0, N, (kt + 1) * BK, K, rb);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      // rows ty*4..+3 and 64+ty*4..+3 ; cols tx*4..+3 and 64+tx*4..+3 (conflict-free float4 reads)
      const float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[cur][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_slab(As[cur ^ 1], ra);
      store_slab(Bs[cur ^ 1], rb);
    }
    __syncthreads();
  }
  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
    const int64_t orow = map(m);
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + jh * 64 + tx * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (n + j >= N) continue;
        float v = acc[i][jh * 4 + j];
        if (bias) v += bias[n + j];
        if (residual) v += residual[orow * ldc + n + j];
        C[orow * ldc + n + j] = v;
      }
    }
  }
}

}  // namespace phk

using namespace phk;

extern "C" int phk_gemm_f32(const float* A, int64_t lda, const float* W, int64_t ldw, float* C, int64_t ldc, int64_t M,
                            int32_t N, int32_t K, const float* bias, const float* residual, int64_t seg_len,
                            int64_t seg_stride, int64_t seg_off, phk_stream_t s) {
  Prof prof_(FAM_GEMM_F32, s, 2.0 * (double)M * N * K);
  PHK_REQUIRE(A && W && C, PHK_E_ARG, "phk_gemm_f32: null pointer");
  PHK_REQUIRE(M >= 0 && N > 0 && K > 0 && lda >= K && ldw >= K && ldc >= N, PHK_E_ARG, "phk_gemm_f32: bad size");
  if (M == 0) return 0;
  const bool aligned = (lda % 4 == 0) && (ldw % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0) &&
                       ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
  dim3 grid((unsigned)((N + BN - 1) / BN), (unsigned)((M + BM - 1) / BM));
  PHK_REQUIRE(grid.y <= 65535, PHK_E_UNSUPPORTED, "phk_gemm_f32: M too large");
  RowMap map{seg_len, seg_stride, seg_off};
  // residual shares C's leading dimension and row map (in-place `x = f(x) + x`, attention.py:323-330)
  if (aligned) PHK_CUDA(launch_pdl(gemm_f32_kernel<true>, dim3(grid), dim3(THREADS), (size_t)(0), to_stream(s), A, lda, W, ldw, C, ldc, M, N, K, bias, residual, map));
  else PHK_CUDA(launch_pdl(gemm_f32_kernel<false>, dim3(grid), dim3(THREADS), (size_t)(0), to_stream(s), A, lda, W, ldw, C, ldc, M, N, K, bias, residual, map));
  PHK_LAUNCH_CHECK();
  return 0;
}
