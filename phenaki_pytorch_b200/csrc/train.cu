// Training step of MaskGit / TokenCritic (SURVEY 8f-2): forward with saved activations, loss, and the hand-written
// backward, fp32 (parity mode).  Reference: Phenaki.forward (phenaki_pytorch.py:562-687) -> MaskGit.forward (:163-213) /
// TokenCritic.forward (:265-302) -> Transformer (attention.py:311-332) under torch autograd.
//
//   phk_maskgit_train_step = embed -> [PEG, self-attn, cross-attn, FF] x depth -> norm_out -> head
//                            -> masked cross entropy (MaskGit, :636-640) | BCE with logits (critic, :672-675)
//                            -> d loss / d every parameter, written into a gradient table of the same layout as the
//                               weight table (the caller zero-fills it; every kernel below ACCUMULATES).
//
// The forward half reuses the library's verified fp32 building blocks (phk_layernorm, phk_gemm_f32, phk_attention,
// phk_peg3d, phk_geglu, phk_token_embed, phk_cpb_bias) and keeps every layer's activations.  The backward kernels are
// deliberately plain (one warp per row, coalesced, no tensor cores): this is the parity path that pins the gradient
// math against the reference's autograd; every formula is restated on the CPU in tests/train_mirror.py and checked
// against the reference there.  In bf16 mode the products run on the tensor-core GEMM instead (see below).
// With dropout (phk_dropout_t) the masks are regenerated from Philox counters wherever they are needed, never stored.
// Checked against the reference's gradients on the CPU by tests/cuda_emu (this very source, g++-compiled) and on the GPU
// by tests/test_gpu_train.py.
#include "phk_common.cuh"
// the kernels of this file are ordinary stream-ordered launches (they do not use programmatic dependent launch)
#define PHK_KERNEL_LAUNCH(kernel, grid, block, smem, st, ...) PHK_CUDA(launch_plain(kernel, grid, block, smem, st, __VA_ARGS__))
#include <cstring>
#include <new>

namespace phk {
namespace {

constexpr float kLnEps = 1e-5f;
constexpr float kL2Eps = 1e-12f;

// ------------------------------------------------------------------------------------------------------------------
// Generic strided fp32 GEMM for the backward products:  C[m, n] (+)= sum_k A(m,k) * B(k,n)
//   A(m,k) = A[m*sam + k*sak],  B(k,n) = B[k*sbk + n*sbn],  C row-major with leading dimension ldc.
//   dgrad  dX[M,K'] = dY[M,N'] . W[N',K']   : sam=N', sak=1, sbk=K', sbn=1
//   wgrad  dW[N',K'] = dY^T . X             : A(m,k)=dY[k*N'+m] (sam=1, sak=N'), B(k,n)=X[k*K'+n] (sbk=K', sbn=1)
// 64x64x16 CTA tile, 256 threads, 4x4 register tile.  Deterministic (no split-K).
// ------------------------------------------------------------------------------------------------------------------
constexpr int GB = 64, GK = 16;

// blockIdx.z = z selects one product of a batch: operand X starts at X + (z / div) * x_outer + (z % div) * x_inner
// (two levels, e.g. (sequence, head) over a token-major [b, n, heads * dim_head] tensor); {1, 1, 0...} = one product
struct GemmBatch {
  int count, div; int64_t a_outer, a_inner, b_outer, b_inner, c_outer, c_inner;
  int k_total;  // > 0: split-K -- batch z multiplies the K range [z * K, min((z + 1) * K, k_total)) (atomic accumulation)
};

__global__ void __launch_bounds__(256) sgemm_strided_kernel(const float* __restrict__ A, int64_t sam, int64_t sak,
                                                            const float* __restrict__ B, int64_t sbk, int64_t sbn,
                                                            float* __restrict__ C, int64_t ldc, int M, int N, int K,
                                                            int accumulate, GemmBatch gb) {
  __shared__ float As[GK][GB + 1];
  __shared__ float Bs[GK][GB + 1];
  {
    const int z = blockIdx.z, zo = z / gb.div, zi = z - zo * gb.div;
    A += zo * gb.a_outer + zi * gb.a_inner;
    B += zo * gb.b_outer + zi * gb.b_inner;
    C += zo * gb.c_outer + zi * gb.c_inner;
  }
  if (gb.k_total > 0) {  // split-K slice of this batch entry
    const int left = gb.k_total - (int)blockIdx.z * K;
    K = left < K ? left : K;
    if (K <= 0) return;
  }
  const int m0 = blockIdx.y * GB, n0 = blockIdx.x * GB;
  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;
  const bool a_kfast = sak == 1;   // which index runs fastest in memory -> which index consecutive threads take
  const bool b_kfast = sbk == 1;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += GK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int mm, kk;
      if (a_kfast) { kk = t & 15; mm = (t >> 4) + 16 * i; } else { mm = t & 63; kk = (t >> 6) + 4 * i; }
      const int m = m0 + mm, k = k0 + kk;
      As[kk][mm] = (m < M && k < K) ? A[(int64_t)m * sam + (int64_t)k * sak] : 0.f;
      int nn, k2;
      if (b_kfast) { k2 = t & 15; nn = (t >> 4) + 16 * i; } else { nn = t & 63; k2 = (t >> 6) + 4 * i; }
      const int n = n0 + nn, kb = k0 + k2;
      Bs[k2][nn] = (n < N && kb < K) ? B[(int64_t)kb * sbk + (int64_t)n * sbn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[k][ty * 4 + i]; b[i] = Bs[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float* c = C + (int64_t)m * ldc + n;
      if (accumulate == 2) atomicAdd(c, acc[i][j]);  // split-K partial sums
      else *c = accumulate ? *c + acc[i][j] : acc[i][j];
    }
  }
}

#ifndef PHK_CUDA_EMU
// The same batched product on warp-level tensor-core MMAs (bf16 training mode: the attention-backward contractions dP, dq,
// dk, dv -- everything but the score recomputation, whose softmax needs fp32-grade logits).  fp32 operands with arbitrary
// strides are converted to bf16 on their way into shared memory (A as [m][k], B as [n][k], 80-byte rows: 16-byte aligned,
// conflict-free ldmatrix), fp32 accumulation, the SIMT kernel's accumulate modes.  64 x 64 tile per CTA, 8 warps of 16 x 32.
constexpr int HK = 32, HLD = HK + 8;
__device__ __forceinline__ void t_ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void t_mma_bf16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(256, 3) hgemm_strided_kernel(const float* __restrict__ A, int64_t sam, int64_t sak,
                                                            const float* __restrict__ B, int64_t sbk, int64_t sbn,
                                                            float* __restrict__ C, int64_t ldc, int M, int N, int K,
                                                            int accumulate, GemmBatch gb) {
  __shared__ __align__(16) __nv_bfloat16 As[GB][HLD];
  __shared__ __align__(16) __nv_bfloat16 Bs[GB][HLD];
  {
    const int z = blockIdx.z, zo = z / gb.div, zi = z - zo * gb.div;
    A += zo * gb.a_outer + zi * gb.a_inner;
    B += zo * gb.b_outer + zi * gb.b_inner;
    C += zo * gb.c_outer + zi * gb.c_inner;
  }
  if (gb.k_total > 0) {
    const int left = gb.k_total - (int)blockIdx.z * K;
    K = left < K ? left : K;
    if (K <= 0) return;
  }
  const int m0 = blockIdx.y * GB, n0 = blockIdx.x * GB;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int wm = (w & 3) * 16, wn = (w >> 2) * 32;  // this warp's 16 x 32 corner of the tile
  const bool a_kfast = sak == 1, b_kfast = sbk == 1;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += HK) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {  // 64 x 32 elements per operand, 8 per thread; consecutive threads along the contiguous index
      int mm, kk;
      if (a_kfast) { kk = t & 31; mm = (t >> 5) + 8 * i; } else { mm = t & 63; kk = (t >> 6) + 4 * i; }
      const int m = m0 + mm, k = k0 + kk;
      As[mm][kk] = __float2bfloat16_rn((m < M && k < K) ? A[(int64_t)m * sam + (int64_t)k * sak] : 0.f);
      int nn, k2;
      if (b_kfast) { k2 = t & 31; nn = (t >> 5) + 8 * i; } else { nn = t & 63; k2 = (t >> 6) + 4 * i; }
      const int n = n0 + nn, kb = k0 + k2;
      Bs[nn][k2] = __float2bfloat16_rn((n < N && kb < K) ? B[(int64_t)kb * sbk + (int64_t)n * sbn] : 0.f);
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < HK / 16; ++ks) {
      uint32_t a[4];
      t_ldmatrix_x4(a, &As[wm + (lane & 7) + 8 * ((lane >> 3) & 1)][ks * 16 + 8 * (lane >> 4)]);
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        uint32_t b[4];
        t_ldmatrix_x4(b, &Bs[wn + (lane & 7) + 8 * (lane >> 4) + 16 * np][ks * 16 + 8 * ((lane >> 3) & 1)]);
        t_mma_bf16_16816(acc[2 * np], a, b[0], b[1]);
        t_mma_bf16_16816(acc[2 * np + 1], a, b[2], b[3]);
      }
    }
    __syncthreads();
  }
  const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int m = m0 + wm + gq + 8 * (e >> 1), n = n0 + wn + nt * 8 + 2 * tq + (e & 1);
      if (m >= M || n >= N) continue;
      float* c = C + (int64_t)m * ldc + n;
      if (accumulate == 2) atomicAdd(c, acc[nt][e]);
      else *c = accumulate ? *c + acc[nt][e] : acc[nt][e];
    }
}
#endif

int sgemm_batched(const float* A, int64_t sam, int64_t sak, const float* B, int64_t sbk, int64_t sbn, float* C, int64_t ldc,
                  int64_t M, int64_t N, int64_t K, int accumulate, const GemmBatch& gb, cudaStream_t st, bool bf16_products = false) {
  PHK_REQUIRE(A && B && C && M > 0 && N > 0 && K > 0, PHK_E_ARG, "train: bad GEMM arguments");
  PHK_REQUIRE(M < (1LL << 31) && N < (1LL << 31) && K < (1LL << 31), PHK_E_UNSUPPORTED, "train: GEMM too large");
  PHK_REQUIRE(gb.count >= 1 && gb.count <= 65535 && gb.div >= 1, PHK_E_UNSUPPORTED, "train: GEMM batch too large");
  dim3 grid((unsigned)((N + GB - 1) / GB), (unsigned)((M + GB - 1) / GB), (unsigned)gb.count);
  PHK_REQUIRE(grid.y <= 65535, PHK_E_UNSUPPORTED, "train: GEMM M too large");
#ifndef PHK_CUDA_EMU
  if (bf16_products) {
    PHK_KERNEL_LAUNCH(hgemm_strided_kernel, dim3(grid), dim3(256), (size_t)(0), st, A, sam, sak, B, sbk, sbn, C, ldc, (int)M, (int)N, (int)K, accumulate, gb);
    PHK_LAUNCH_CHECK();
    return 0;
  }
#endif
  (void)bf16_products;
  PHK_KERNEL_LAUNCH(sgemm_strided_kernel, dim3(grid), dim3(256), (size_t)(0), st, A, sam, sak, B, sbk, sbn, C, ldc, (int)M, (int)N, (int)K, accumulate, gb);
  PHK_LAUNCH_CHECK();
  return 0;
}
int sgemm(const float* A, int64_t sam, int64_t sak, const float* B, int64_t sbk, int64_t sbn, float* C, int64_t ldc,
          int64_t M, int64_t N, int64_t K, int accumulate, cudaStream_t st) {
  return sgemm_batched(A, sam, sak, B, sbk, sbn, C, ldc, M, N, K, accumulate, GemmBatch{1, 1, 0, 0, 0, 0, 0, 0, 0}, st);
}
// dX[M,K] (+)= dY[M,N] . W[N,K]        (nn.Linear dgrad)
int dgrad(const float* dY, const float* W, float* dX, int64_t M, int64_t N, int64_t K, int accumulate, cudaStream_t st) {
  return sgemm(dY, N, 1, W, K, 1, dX, K, M, K, N, accumulate, st);
}
// dW[N,K] += dY[M,N]^T . X[M,K]        (nn.Linear wgrad)
int wgrad(const float* dY, const float* X, float* dW, int64_t M, int64_t N, int64_t K, cudaStream_t st) {
  // small weight, long reduction (the position-bias MLP over thousands of coordinate deltas: [64 x 64] += over 3825 rows
  // was ONE CTA for 0.3 ms): split the reduction over the batch dimension, partial sums meet in dW through atomics
  if (N * K <= 4 * GB * GB && M >= 1024) {
    const int64_t chunk = 256;
    const int parts = (int)((M + chunk - 1) / chunk);
    const GemmBatch gb{parts, 1, chunk * N, 0, chunk * K, 0, 0, 0, (int)M};
    return sgemm_batched(dY, 1, N, X, K, 1, dW, K, N, K, chunk, 2, gb, st);
  }
  return sgemm(dY, 1, N, X, K, 1, dW, K, N, K, M, 1, st);
}
inline unsigned ew_grid_fwd(int64_t total) {
  const int64_t b = (total + 255) / 256;
  return (unsigned)(b < 1 ? 1 : (b > kNumSMs * 16 ? kNumSMs * 16 : b));
}

// out[c] += sum_r x[r, c]   (bias gradients); grid (ceil(C/256), row chunks), atomics across chunks
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, int64_t rows, int cols, int64_t ld,
                                                     float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const int64_t per = (rows + gridDim.y - 1) / gridDim.y;
  const int64_t r0 = (int64_t)blockIdx.y * per, r1 = r0 + per < rows ? r0 + per : rows;
  float a = 0.f;
  for (int64_t r = r0; r < r1; ++r) a += x[r * ld + c];
  if (r1 > r0) atomicAdd(out + c, a);
}
int colsum(const float* x, int64_t rows, int cols, int64_t ld, float* out, cudaStream_t st) {
  int chunks = (int)((rows + 63) / 64);
  if (chunks > 64) chunks = 64;
  if (chunks < 1) chunks = 1;
  PHK_KERNEL_LAUNCH(colsum_kernel, dim3((unsigned)((cols + 255) / 256), (unsigned)chunks), dim3(256), (size_t)(0), st, x, rows, cols, ld, out);
  PHK_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// bf16 mode (PHK_PREC_BF16): the three products of every nn.Linear run on the wgmma GEMM of gemm_wgmma.cu
// (C = A.W^T, bf16 operands K-major, fp32 accumulate -- the dtype flow of torch.autocast(bfloat16)); the operands are
// converted on the fly from the fp32 activations / master weights:
//   forward  Y[M,N]  = X.W^T          A = bf16(X) [M,K]        W = bf16(W) [N,K]
//   dgrad    dX[M,K] (+)= dY.W        A = bf16(dY) [M,N]       W = bf16(W)^T [K,N]
//   wgrad    dW[N,K] += dY^T.X        A = bf16(dY)^T [N,M]     W = bf16(X)^T [K,M]
// Leading dimensions are padded to a multiple of 8 elements (TMA); the tensor maps stop at the true extent, so the
// padding is never read.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cast_bf16_kernel(const float* __restrict__ src, int64_t rows, int cols,
                                                        __nv_bfloat16* __restrict__ dst, int64_t ldd) {
  const int64_t total = rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cols;
    dst[r * ldd + (i - r * cols)] = __float2bfloat16_rn(src[i]);
  }
}
// dst[c, r] = bf16(src[r, c]); 32 x 32 tiles through shared memory so that both sides are coalesced
__global__ void __launch_bounds__(256) cast_transpose_bf16_kernel(const float* __restrict__ src, int64_t rows, int cols,
                                                                  __nv_bfloat16* __restrict__ dst, int64_t ldd) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t r0 = (int64_t)blockIdx.y * 32;
  const int c0 = blockIdx.x * 32;
  for (int i = ty; i < 32; i += 8) {
    const int64_t r = r0 + i;
    const int c = c0 + tx;
    tile[i][tx] = (r < rows && c < cols) ? src[r * cols + c] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i;
    const int64_t r = r0 + tx;
    if (c < cols && r < rows) dst[(int64_t)c * ldd + r] = __float2bfloat16_rn(tile[tx][i]);
  }
}

struct TcScratch { __nv_bfloat16* a; __nv_bfloat16* b; int64_t elems; };  // two operand buffers of `elems` bf16 each
inline int64_t pad8(int64_t v) { return (v + 7) / 8 * 8; }

int cast_to(const float* src, int64_t rows, int64_t cols, bool transpose, __nv_bfloat16* dst, int64_t cap, int64_t* ld,
            cudaStream_t st) {
  PHK_REQUIRE(rows > 0 && cols > 0 && cols < (1LL << 31), PHK_E_ARG, "train: bad operand shape");
  if (!transpose) {
    *ld = pad8(cols);
    PHK_REQUIRE(rows * *ld <= cap, PHK_E_WORKSPACE, "train: tensor-core operand scratch too small");
    PHK_KERNEL_LAUNCH(cast_bf16_kernel, dim3(ew_grid_fwd(rows * cols)), dim3(256), (size_t)(0), st, src, rows, (int)cols, dst, *ld);
  } else {
    *ld = pad8(rows);
    PHK_REQUIRE(cols * *ld <= cap, PHK_E_WORKSPACE, "train: tensor-core operand scratch too small");
    PHK_REQUIRE((rows + 31) / 32 <= 65535, PHK_E_UNSUPPORTED, "train: operand too tall for the transposing cast");
    PHK_KERNEL_LAUNCH(cast_transpose_bf16_kernel, dim3((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32)), dim3(256), (size_t)(0), st, src, rows, (int)cols, dst, *ld);
  }
  PHK_LAUNCH_CHECK();
  return 0;
}

// Y[M,N] = X[M,K].W[N,K]^T (+bias) (+residual: `residual` must be Y itself, i.e. Y already holds the residual)
int linear_fwd(int prec, const TcScratch& tc, const float* X, const float* W, float* Y, int64_t M, int64_t N, int64_t K,
               const float* bias, const float* residual, phk_stream_t s) {
  if (prec != PHK_PREC_BF16)
    return phk_gemm_f32(X, K, W, K, Y, N, M, (int32_t)N, (int32_t)K, bias, residual, 0, 0, 0, s);
  int64_t lda = 0, ldw = 0;
  PHK_TRY(cast_to(X, M, K, false, tc.a, tc.elems, &lda, to_stream(s)));
  PHK_TRY(cast_to(W, N, K, false, tc.b, tc.elems, &ldw, to_stream(s)));
  if (residual && residual != Y) PHK_CUDA(cudaMemcpyAsync(Y, residual, M * N * 4, cudaMemcpyDeviceToDevice, to_stream(s)));
  return phk_gemm_bf16(tc.a, lda, tc.b, ldw, Y, N, M, (int32_t)N, (int32_t)K, bias, residual ? Y : nullptr, 0, 0, 0, 0, s);
}
// dX[M,K] (+)= dY[M,N] . W[N,K]
int dgrad_p(int prec, const TcScratch& tc, const float* dY, const float* W, float* dX, int64_t M, int64_t N, int64_t K,
            int accumulate, phk_stream_t s) {
  if (prec != PHK_PREC_BF16) return dgrad(dY, W, dX, M, N, K, accumulate, to_stream(s));
  int64_t lda = 0, ldw = 0;
  PHK_TRY(cast_to(dY, M, N, false, tc.a, tc.elems, &lda, to_stream(s)));
  PHK_TRY(cast_to(W, N, K, true, tc.b, tc.elems, &ldw, to_stream(s)));  // W^T [K, N]
  return phk_gemm_bf16(tc.a, lda, tc.b, ldw, dX, K, M, (int32_t)K, (int32_t)N, nullptr, accumulate ? dX : nullptr, 0, 0, 0, 0, s);
}
// dW[N,K] += dY[M,N]^T . X[M,K]
int wgrad_p(int prec, const TcScratch& tc, const float* dY, const float* X, float* dW, int64_t M, int64_t N, int64_t K,
            phk_stream_t s) {
  if (prec != PHK_PREC_BF16) return wgrad(dY, X, dW, M, N, K, to_stream(s));
  int64_t lda = 0, ldw = 0;
  PHK_TRY(cast_to(dY, M, N, true, tc.a, tc.elems, &lda, to_stream(s)));  // dY^T [N, M]
  PHK_TRY(cast_to(X, M, K, true, tc.b, tc.elems, &ldw, to_stream(s)));   // X^T  [K, M]
  return phk_gemm_bf16(tc.a, lda, tc.b, ldw, dW, K, N, (int32_t)K, (int32_t)M, nullptr, dW, 0, 0, 0, 0, s);
}

// ------------------------------------------------------------------------------------------------------------------
// LayerNorm backward (tests/train_mirror.py::ln_bwd).  One warp per row:
//   xhat = (x - mean) * rstd ; dxh = dy * g ; dx (+)= rstd * (dxh - mean(dxh) - xhat * mean(dxh * xhat))
// stats[r] = (mean, rstd) is kept for the column kernel:  dgamma[c] += sum_r dy * xhat ; dbeta[c] += sum_r dy
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ln_bwd_dx_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                        const float* __restrict__ dy, float* __restrict__ dx,
                                                        float2* __restrict__ stats, int64_t rows, int dim,
                                                        int accumulate) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * dim;
  const float* dyr = dy + row * dim;
  float s = 0.f;
  for (int c = lane; c < dim; c += 32) s += xr[c];
  const float mean = warp_sum(s) / (float)dim;
  float q = 0.f;
  for (int c = lane; c < dim; c += 32) { const float d = xr[c] - mean; q += d * d; }
  const float rstd = rsqrtf(warp_sum(q) / (float)dim + kLnEps);
  float s1 = 0.f, s2 = 0.f;
  for (int c = lane; c < dim; c += 32) {
    const float dxh = dyr[c] * g[c];
    s1 += dxh;
    s2 += dxh * (xr[c] - mean) * rstd;
  }
  const float c1 = warp_sum(s1) / (float)dim, c2 = warp_sum(s2) / (float)dim;
  if (dx) {
    float* dxr = dx + row * dim;
    for (int c = lane; c < dim; c += 32) {
      const float xh = (xr[c] - mean) * rstd;
      const float v = rstd * (dyr[c] * g[c] - c1 - xh * c2);
      dxr[c] = accumulate ? dxr[c] + v : v;
    }
  }
  if (lane == 0) stats[row] = make_float2(mean, rstd);
}

__global__ void __launch_bounds__(256) ln_bwd_dgb_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                         const float2* __restrict__ stats, int64_t rows, int dim,
                                                         float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= dim) return;
  const int64_t per = (rows + gridDim.y - 1) / gridDim.y;
  const int64_t r0 = (int64_t)blockIdx.y * per, r1 = r0 + per < rows ? r0 + per : rows;
  float ag = 0.f, ab = 0.f;
  for (int64_t r = r0; r < r1; ++r) {
    const float2 st = stats[r];
    const float d = dy[r * dim + c];
    ag += d * (x[r * dim + c] - st.x) * st.y;
    ab += d;
  }
  if (r1 > r0) {
    atomicAdd(dgamma + c, ag);
    if (dbeta) atomicAdd(dbeta + c, ab);
  }
}

// dx (+)= LN_bwd(x; g)(dy); dgamma += ..; dbeta += .. (dbeta NULL: the custom LayerNorm's beta is a buffer)
int ln_backward(const float* x, const float* g, const float* dy, float* dx, int accumulate, float* dgamma, float* dbeta,
                float2* stats, int64_t rows, int dim, cudaStream_t st) {
  PHK_KERNEL_LAUNCH(ln_bwd_dx_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), (size_t)(0), st, x, g, dy, dx, stats, rows, dim, accumulate);
  PHK_LAUNCH_CHECK();
  int chunks = (int)((rows + 63) / 64);
  if (chunks > 64) chunks = 64;
  PHK_KERNEL_LAUNCH(ln_bwd_dgb_kernel, dim3((unsigned)((dim + 255) / 256), (unsigned)chunks), dim3(256), (size_t)(0), st, x, dy, stats, rows, dim, dgamma,
                                                                                           dbeta);
  PHK_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// Dropout (include/phk.h, phk_dropout_t): element e of a site is kept iff u(base + e/4, word e % 4) >= p and then scaled
// by 1/(1 - p); u is the sampling noise's uniform of that Philox4x32-7 block.  p == 0: the site is off.
// ------------------------------------------------------------------------------------------------------------------
struct DropSite { float p, scale; uint32_t k0, k1; uint64_t base; };

__device__ __forceinline__ float drop_factor(const DropSite& d, uint64_t e) {
  const uint64_t c = d.base + (e >> 2);
  uint32_t r[4];
  philox4x32<kNoiseRounds>((uint32_t)c, (uint32_t)(c >> 32), 0u, 0u, d.k0, d.k1, r);
  const uint32_t k = (uint32_t)(e & 3);
  const uint32_t w = k == 0 ? r[0] : (k == 1 ? r[1] : (k == 2 ? r[2] : r[3]));
  const float u = (float)(2u * (w >> 9) + 1u) * (1.0f / 16777216.0f);  // exact: 2 (w >> 9) + 1 < 2^24
  return u >= d.p ? d.scale : 0.f;                                      // p = 1 keeps nothing (u < 1): zeros, not NaN
}

// g = gelu(gate) * val * M / (1 - p): GEGLU followed by the FF dropout (attention.py:51), the dropped g is what W2 reads
__global__ void geglu_dropout_kernel(const float* __restrict__ h, float* __restrict__ g, int64_t rows, int inner,
                                     DropSite d) {
  const int64_t total = rows * inner;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / inner;
    const int j = (int)(i - r * inner);
    const float m = drop_factor(d, (uint64_t)i);
    g[i] = m != 0.f ? gelu_erf(h[r * 2 * inner + inner + j]) * h[r * 2 * inner + j] * m : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// GEGLU backward (attention.py:40-43; mirror geglu_bwd): h = [val | gate], g = gelu_erf(gate) * val
//   dval = dg * gelu(gate) ; dgate = dg * val * (Phi(gate) + gate * phi(gate))
// With FF dropout (d.p > 0) the incoming gradient is that of the dropped g: dg is first multiplied by M / (1 - p).
// ------------------------------------------------------------------------------------------------------------------
__global__ void geglu_bwd_kernel(const float* __restrict__ h, const float* __restrict__ dg, float* __restrict__ dh,
                                 int64_t rows, int inner, DropSite drop) {
  const int64_t total = rows * inner;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / inner;
    const int j = (int)(i - r * inner);
    const float val = h[r * 2 * inner + j], gate = h[r * 2 * inner + inner + j];
    const float d = drop.p > 0.f ? dg[i] * drop_factor(drop, (uint64_t)i) : dg[i];
    const float cdf = 0.5f * (1.0f + erff(gate * 0.70710678118654752440f));
    const float pdf = expf(-0.5f * gate * gate) * 0.39894228040143267794f;
    dh[r * 2 * inner + j] = d * gate * cdf;
    dh[r * 2 * inner + inner + j] = d * val * (cdf + gate * pdf);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Attention backward (attention.py:146-181; mirror attn_bwd).  Sequences are (b, n) rows of q [b*n, I] and
// (b, m) rows of kv [b*m, 2I]; nkt = nnull + m keys per (sequence, head).
//   prep : qh = l2norm(q) * q_scale, kh = l2norm(k) * k_scale, vv   -> head-major [b, H, n|nkt, dh]
//   S, dP: qh.kh^T and dO.vv^T as two batched register-tiled products                       -> [b, H, n, nkt]
//   probs: P = softmax(8 S + bias, masks) ; dS = P * (dP - sum_j P dP), in place, rows coalesced
//   dq   : dqh = 8 dS.kh -> back through scale and l2norm -> dq [b*n, I], dq_scale
//   dkv  : dkh = 8 dS^T.qh, dvv = P^T.dO -> back through scale and l2norm -> dkv [b*m, 2I], dnull_kv, dk_scale
// ------------------------------------------------------------------------------------------------------------------
struct AttnBwdGeom { int b, H, n, m, nnull, dh; };

__device__ __forceinline__ const float* key_row(const float* kv, const float* null_kv, const AttnBwdGeom& g, int bi, int h,
                                                int j, bool value) {
  const int I = g.H * g.dh;
  if (j < g.nnull) return null_kv + ((int64_t)h * 2 * g.nnull + 2 * j + (value ? 1 : 0)) * g.dh;  // 'h (n r) d' (:148)
  return kv + ((int64_t)bi * g.m + (j - g.nnull)) * 2 * I + (value ? I : 0) + (int64_t)h * g.dh;
}

// one warp per (sequence, head, row): rows [0, n) are queries, rows [n, n + nkt) are keys
__global__ void __launch_bounds__(256) attn_bwd_prep_kernel(const float* __restrict__ q, const float* __restrict__ kv,
                                                            const float* __restrict__ null_kv,
                                                            const float* __restrict__ q_scale,
                                                            const float* __restrict__ k_scale, float* __restrict__ qh,
                                                            float* __restrict__ kh, float* __restrict__ vv,
                                                            AttnBwdGeom g) {
  const int lane = threadIdx.x & 31;
  const int nkt = g.nnull + g.m, per = g.n + nkt;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= (int64_t)g.b * g.H * per) return;
  const int r = (int)(w % per);
  const int h = (int)((w / per) % g.H);
  const int bi = (int)(w / ((int64_t)per * g.H));
  const int I = g.H * g.dh;
  const bool is_q = r < g.n;
  const float* src = is_q ? q + ((int64_t)bi * g.n + r) * I + (int64_t)h * g.dh : key_row(kv, null_kv, g, bi, h, r - g.n, false);
  float ss = 0.f;
  for (int d = lane; d < g.dh; d += 32) ss += src[d] * src[d];
  const float nrm = fmaxf(sqrtf(warp_sum(ss)), kL2Eps);
  if (is_q) {
    float* dst = qh + (((int64_t)bi * g.H + h) * g.n + r) * g.dh;
    for (int d = lane; d < g.dh; d += 32) dst[d] = (src[d] / nrm) * q_scale[d];
  } else {
    const int j = r - g.n;
    float* dst = kh + (((int64_t)bi * g.H + h) * nkt + j) * g.dh;
    float* dv = vv + (((int64_t)bi * g.H + h) * nkt + j) * g.dh;
    const float* vs = key_row(kv, null_kv, g, bi, h, j, true);
    for (int d = lane; d < g.dh; d += 32) { dst[d] = (src[d] / nrm) * k_scale[d]; dv[d] = vs[d]; }
  }
}

// Forward with attention dropout, one warp per (sequence, head, query).  In: P holds the raw products qh.kh.
// Out (in place): P = softmax(8 qh.kh + bias, masks) * M / (1 - p), element e = row * nkt + j of the site.
__global__ void __launch_bounds__(256) attn_fwd_softmax_dropout_kernel(const float* __restrict__ bias,
                                                                       const uint8_t* __restrict__ key_mask,
                                                                       float* __restrict__ P, AttnBwdGeom g, DropSite d) {
  const int lane = threadIdx.x & 31;
  const int nkt = g.nnull + g.m;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= (int64_t)g.b * g.H * g.n) return;
  const int i = (int)(w % g.n);
  const int h = (int)((w / g.n) % g.H);
  const int bi = (int)(w / ((int64_t)g.n * g.H));
  float* Pr = P + w * nkt;
  float mx = -FLT_MAX;
  for (int j = lane; j < nkt; j += 32) {
    float s = Pr[j] * 8.0f;
    if (bias && j >= g.nnull) s += bias[((int64_t)h * g.n + i) * g.m + (j - g.nnull)];
    if (key_mask && j >= g.nnull && !key_mask[(int64_t)bi * g.m + (j - g.nnull)]) s = -FLT_MAX;
    Pr[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < nkt; j += 32) { const float e = expf(Pr[j] - mx); Pr[j] = e; sum += e; }
  sum = warp_sum(sum);
  const float inv = 1.0f / sum;
  for (int j = lane; j < nkt; j += 32) {
    const float m = drop_factor(d, (uint64_t)w * nkt + j);
    Pr[j] = m != 0.f ? Pr[j] * inv * m : 0.f;
  }
}

// one warp per (sequence, head, query).  In: P holds the raw products qh.kh (batched GEMM), dS holds dP = dO.vv.
// Out (in place): P = softmax(8 qh.kh + bias, masks), dS = P * (dP - sum_j P dP).  Rows are contiguous: coalesced.
// With attention dropout (d.p > 0) dS holds the gradient of the DROPPED probabilities: dP = dS * M / (1 - p) enters the
// softmax backward, which differentiates the undropped P; P is then overwritten by the dropped P that the forward
// multiplied V with (what dV = P^T.dO needs).
__global__ void __launch_bounds__(256) attn_bwd_softmax_kernel(const float* __restrict__ bias,
                                                               const uint8_t* __restrict__ key_mask, float* __restrict__ P,
                                                               float* __restrict__ dS, AttnBwdGeom g, DropSite d) {
  const int lane = threadIdx.x & 31;
  const int nkt = g.nnull + g.m;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= (int64_t)g.b * g.H * g.n) return;
  const int i = (int)(w % g.n);
  const int h = (int)((w / g.n) % g.H);
  const int bi = (int)(w / ((int64_t)g.n * g.H));
  float* Pr = P + w * nkt;    // w = (bi * H + h) * n + i
  float* dSr = dS + w * nkt;
  float mx = -FLT_MAX;
  for (int j = lane; j < nkt; j += 32) {
    float s = Pr[j] * 8.0f;                                                                // scale (attention.py:100)
    if (bias && j >= g.nnull) s += bias[((int64_t)h * g.n + i) * g.m + (j - g.nnull)];    // never covers null keys (:162)
    if (key_mask && j >= g.nnull && !key_mask[(int64_t)bi * g.m + (j - g.nnull)]) s = -FLT_MAX;  // (:166-167)
    Pr[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < nkt; j += 32) { const float e = expf(Pr[j] - mx); Pr[j] = e; sum += e; }
  sum = warp_sum(sum);
  const float inv = 1.0f / sum;
  float dot = 0.f;
  if (d.p > 0.f) {
    for (int j = lane; j < nkt; j += 32) {
      const float p = Pr[j] * inv;
      const float dp = dSr[j] * drop_factor(d, (uint64_t)w * nkt + j);
      Pr[j] = p; dSr[j] = dp; dot += p * dp;
    }
    dot = warp_sum(dot);
    for (int j = lane; j < nkt; j += 32) {
      const float m = drop_factor(d, (uint64_t)w * nkt + j);
      dSr[j] = Pr[j] * (dSr[j] - dot);
      Pr[j] = m != 0.f ? Pr[j] * m : 0.f;
    }
    return;
  }
  for (int j = lane; j < nkt; j += 32) { const float p = Pr[j] * inv; Pr[j] = p; dot += p * dSr[j]; }
  dot = warp_sum(dot);
  for (int j = lane; j < nkt; j += 32) dSr[j] = Pr[j] * (dSr[j] - dot);
}

// back through `hat = (raw / max(|raw|, eps)) * scale` for one dh-vector held as DPL values per lane:
//   dscale[d] += dhat[d] * u[d] ; g = dhat * scale ; draw = (g - u * (u.g)) / r
template <int DPL>
__device__ __forceinline__ void l2norm_scale_bwd(const float* __restrict__ raw, const float* __restrict__ scale,
                                                 const float (&dhat)[DPL], int dh, int lane, float (&draw)[DPL],
                                                 float (&dsc)[DPL]) {
  float x[DPL], ss = 0.f;
#pragma unroll
  for (int c = 0; c < DPL; ++c) { const int d = lane + 32 * c; x[c] = d < dh ? raw[d] : 0.f; ss += x[c] * x[c]; }
  const float r = fmaxf(sqrtf(warp_sum(ss)), kL2Eps);
  float ug = 0.f, gv[DPL], u[DPL];
#pragma unroll
  for (int c = 0; c < DPL; ++c) {
    const int d = lane + 32 * c;
    u[c] = x[c] / r;
    gv[c] = d < dh ? dhat[c] * scale[d] : 0.f;
    dsc[c] = dhat[c] * u[c];
    ug += u[c] * gv[c];
  }
  ug = warp_sum(ug);
#pragma unroll
  for (int c = 0; c < DPL; ++c) draw[c] = (gv[c] - u[c] * ug) / r;
}

constexpr int kDPL = 4;  // dim_head <= 128

// one warp per (sequence, head, query): dqh = 8 * sum_j dS[i,j] kh[j,:]; 8 warps per CTA share one dq_scale reduction
// `pre` (optional): dS.kh already computed as a batched register-tiled product [b*H, n, dh] (long sequences: the warp-per-
// row loop below re-reads the whole key block per query)
__global__ void __launch_bounds__(256) attn_bwd_dq_kernel(const float* __restrict__ q, const float* __restrict__ kh,
                                                          const float* __restrict__ dS, const float* __restrict__ q_scale,
                                                          float* __restrict__ dq, float* __restrict__ dq_scale,
                                                          const float* __restrict__ pre, AttnBwdGeom g) {
  __shared__ float red[8][32 * kDPL];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nkt = g.nnull + g.m;
  const int I = g.H * g.dh;
  const int64_t w = (int64_t)blockIdx.x * 8 + wid;
  const bool active = w < (int64_t)g.b * g.H * g.n;
  float dsc[kDPL] = {0.f, 0.f, 0.f, 0.f};
  if (active) {
    const int i = (int)(w % g.n);
    const int h = (int)((w / g.n) % g.H);
    const int bi = (int)(w / ((int64_t)g.n * g.H));
    const float* dSr = dS + (((int64_t)bi * g.H + h) * g.n + i) * nkt;
    const float* kb = kh + ((int64_t)bi * g.H + h) * nkt * g.dh;
    float acc[kDPL] = {0.f, 0.f, 0.f, 0.f};
    if (pre) {
#pragma unroll
      for (int c = 0; c < kDPL; ++c) { const int d = lane + 32 * c; if (d < g.dh) acc[c] = pre[w * g.dh + d]; }
    } else {
      for (int j = 0; j < nkt; ++j) {
        const float s = dSr[j];
#pragma unroll
        for (int c = 0; c < kDPL; ++c) { const int d = lane + 32 * c; if (d < g.dh) acc[c] = fmaf(s, kb[(int64_t)j * g.dh + d], acc[c]); }
      }
    }
#pragma unroll
    for (int c = 0; c < kDPL; ++c) acc[c] *= 8.0f;
    const float* raw = q + ((int64_t)bi * g.n + i) * I + (int64_t)h * g.dh;
    float draw[kDPL];
    l2norm_scale_bwd<kDPL>(raw, q_scale, acc, g.dh, lane, draw, dsc);
    float* out = dq + ((int64_t)bi * g.n + i) * I + (int64_t)h * g.dh;
#pragma unroll
    for (int c = 0; c < kDPL; ++c) { const int d = lane + 32 * c; if (d < g.dh) out[d] = draw[c]; }
  }
#pragma unroll
  for (int c = 0; c < kDPL; ++c) red[wid][lane + 32 * c] = dsc[c];
  __syncthreads();
  if (threadIdx.x < g.dh) {
    float a = 0.f;
    for (int k = 0; k < 8; ++k) a += red[k][threadIdx.x];
    atomicAdd(dq_scale + threadIdx.x, a);
  }
}

// one warp per (sequence, head, key j in [0, nkt)): dkh = 8 * sum_i dS[i,j] qh[i,:], dvv = sum_i P[i,j] dO[i,:]
__global__ void __launch_bounds__(256) attn_bwd_dkv_kernel(const float* __restrict__ kv, const float* __restrict__ null_kv,
                                                           const float* __restrict__ qh, const float* __restrict__ dO,
                                                           const float* __restrict__ P, const float* __restrict__ dS,
                                                           const float* __restrict__ k_scale, float* __restrict__ dkv,
                                                           float* __restrict__ dnull_kv, float* __restrict__ dk_scale,
                                                           const float* __restrict__ preK, const float* __restrict__ preV,
                                                           AttnBwdGeom g) {
  __shared__ float red[8][32 * kDPL];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nkt = g.nnull + g.m;
  const int I = g.H * g.dh;
  const int64_t w = (int64_t)blockIdx.x * 8 + wid;
  const bool active = w < (int64_t)g.b * g.H * nkt;
  float dsc[kDPL] = {0.f, 0.f, 0.f, 0.f};
  if (active) {
    const int j = (int)(w % nkt);
    const int h = (int)((w / nkt) % g.H);
    const int bi = (int)(w / ((int64_t)nkt * g.H));
    const float* Pb = P + ((int64_t)bi * g.H + h) * g.n * nkt + j;
    const float* dSb = dS + ((int64_t)bi * g.H + h) * g.n * nkt + j;
    const float* qb = qh + ((int64_t)bi * g.H + h) * g.n * g.dh;
    const float* dob = dO + (int64_t)bi * g.n * I + (int64_t)h * g.dh;
    float ak[kDPL] = {0.f, 0.f, 0.f, 0.f}, av[kDPL] = {0.f, 0.f, 0.f, 0.f};
    if (preK) {  // dS^T.qh and P^T.dO from the batched products [b*H, nkt, dh]
#pragma unroll
      for (int c = 0; c < kDPL; ++c) {
        const int d = lane + 32 * c;
        if (d < g.dh) { ak[c] = preK[w * g.dh + d]; av[c] = preV[w * g.dh + d]; }
      }
    } else {
      for (int i = 0; i < g.n; ++i) {
        const float s = dSb[(int64_t)i * nkt], p = Pb[(int64_t)i * nkt];
#pragma unroll
        for (int c = 0; c < kDPL; ++c) {
          const int d = lane + 32 * c;
          if (d < g.dh) { ak[c] = fmaf(s, qb[(int64_t)i * g.dh + d], ak[c]); av[c] = fmaf(p, dob[(int64_t)i * I + d], av[c]); }
        }
      }
    }
#pragma unroll
    for (int c = 0; c < kDPL; ++c) ak[c] *= 8.0f;
    const float* raw = key_row(kv, null_kv, g, bi, h, j, false);
    float draw[kDPL];
    l2norm_scale_bwd<kDPL>(raw, k_scale, ak, g.dh, lane, draw, dsc);
    if (j < g.nnull) {  // the null keys / values are parameters shared by every sequence: accumulate over the batch
      float* nk = dnull_kv + ((int64_t)h * 2 * g.nnull + 2 * j) * g.dh;
#pragma unroll
      for (int c = 0; c < kDPL; ++c) {
        const int d = lane + 32 * c;
        if (d < g.dh) { atomicAdd(nk + d, draw[c]); atomicAdd(nk + g.dh + d, av[c]); }
      }
    } else {
      float* out = dkv + ((int64_t)bi * g.m + (j - g.nnull)) * 2 * I + (int64_t)h * g.dh;
#pragma unroll
      for (int c = 0; c < kDPL; ++c) { const int d = lane + 32 * c; if (d < g.dh) { out[d] = draw[c]; out[I + d] = av[c]; } }
    }
  }
#pragma unroll
  for (int c = 0; c < kDPL; ++c) red[wid][lane + 32 * c] = dsc[c];
  __syncthreads();
  if (threadIdx.x < g.dh) {
    float a = 0.f;
    for (int k = 0; k < 8; ++k) a += red[k][threadIdx.x];
    atomicAdd(dk_scale + threadIdx.x, a);
  }
}

// dbias[h, i, j] += sum_b dS[b, h, i, nnull + j]   (self-attention position bias, shared by batch and layers)
__global__ void attn_bwd_dbias_kernel(const float* __restrict__ dS, float* __restrict__ dbias, AttnBwdGeom g) {
  const int nkt = g.nnull + g.m;
  const int64_t total = (int64_t)g.H * g.n * g.m;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx % g.m);
    const int64_t hi = idx / g.m;  // h * n + i
    float a = 0.f;
    for (int bi = 0; bi < g.b; ++bi) a += dS[((int64_t)bi * g.H * g.n + hi) * nkt + g.nnull + j];
    dbias[idx] += a;
  }
}

struct AttnBwdBufs { float *qh, *kh, *vv, *P, *dS; };

int64_t attn_bwd_scratch_floats(int b, int H, int n, int nkt, int dh) {
  // qh, kh, vv, P, dS + the batched-product outputs dS.kh [n, dh], dS^T.qh and P^T.dO [nkt, dh]
  return (int64_t)b * H * (2 * (int64_t)n * dh + 4 * (int64_t)nkt * dh + 2 * (int64_t)n * nkt) + 64;
}

// q [b*n, I], kv [b*m, 2I], dO [b*n, I] -> dq [b*n, I], dkv [b*m, 2I]; parameter gradients accumulate
int attention_backward(const float* q, const float* kv, const phk_attn_t& A, const phk_attn_t& G, const float* bias,
                       const uint8_t* key_mask, const float* dO, float* dq, float* dkv, float* dbias,
                       const AttnBwdGeom& g, float* scratch, cudaStream_t st, bool bf16_products, const DropSite& drop) {
  PHK_REQUIRE(g.dh <= 32 * kDPL, PHK_E_UNSUPPORTED, "train: dim_head > 128");
  PHK_REQUIRE(g.nnull == 0 || (A.null_kv && G.null_kv), PHK_E_ARG, "train: null_kv (gradient) missing");
  const int nkt = g.nnull + g.m;
  const int64_t bh = (int64_t)g.b * g.H;
  AttnBwdBufs B;
  B.qh = scratch;
  B.kh = B.qh + bh * g.n * g.dh;
  B.vv = B.kh + bh * nkt * g.dh;
  B.P = B.vv + bh * nkt * g.dh;
  B.dS = B.P + bh * g.n * nkt;
  const int64_t prep_warps = bh * (g.n + nkt);
  PHK_KERNEL_LAUNCH(attn_bwd_prep_kernel, dim3((unsigned)((prep_warps + 7) / 8)), dim3(256), (size_t)(0), st, q, kv, A.null_kv, A.q_scale, A.k_scale, B.qh, B.kh,
                                                                        B.vv, g);
  PHK_LAUNCH_CHECK();
  // S = qh.kh^T and dP = dO.vv^T for every (sequence, head): two batched register-tiled products (a warp-per-row dot
  // product would read the key rows with a stride of dim_head floats between lanes)
  const int I = g.H * g.dh;
  const GemmBatch bs{(int)bh, 1, (int64_t)g.n * g.dh, 0, (int64_t)nkt * g.dh, 0, (int64_t)g.n * nkt, 0};
  PHK_TRY(sgemm_batched(B.qh, g.dh, 1, B.kh, 1, g.dh, B.P, nkt, g.n, nkt, g.dh, 0, bs, st));
  const GemmBatch bd{(int)bh, g.H, (int64_t)g.n * I, (int64_t)g.dh, (int64_t)g.H * nkt * g.dh, (int64_t)nkt * g.dh,
                     (int64_t)g.H * g.n * nkt, (int64_t)g.n * nkt};
  PHK_TRY(sgemm_batched(dO, I, 1, B.vv, 1, g.dh, B.dS, nkt, g.n, nkt, g.dh, 0, bd, st, bf16_products));
  PHK_KERNEL_LAUNCH(attn_bwd_softmax_kernel, dim3((unsigned)((bh * g.n + 7) / 8)), dim3(256), (size_t)(0), st, bias, key_mask, B.P, B.dS, g, drop);
  PHK_LAUNCH_CHECK();
  // dq / dk / dv contractions: batched register-tiled products for long sequences (the warp-per-row loops of the two
  // kernels walk a column of dS / P with a stride of nkt floats: 1.5 ms per layer at n = 576), loops for short ones
  float* preQ = nullptr; float* preK = nullptr; float* preV = nullptr;
  if ((int64_t)g.n * nkt >= 64 * 64) {
    preQ = B.dS + bh * g.n * nkt;
    preK = preQ + bh * g.n * g.dh;
    preV = preK + bh * nkt * g.dh;
    const GemmBatch bq{(int)bh, 1, (int64_t)g.n * nkt, 0, (int64_t)nkt * g.dh, 0, (int64_t)g.n * g.dh, 0};
    PHK_TRY(sgemm_batched(B.dS, nkt, 1, B.kh, g.dh, 1, preQ, g.dh, g.n, g.dh, nkt, 0, bq, st, bf16_products));  // dS . kh
    const GemmBatch bk{(int)bh, 1, (int64_t)g.n * nkt, 0, (int64_t)g.n * g.dh, 0, (int64_t)nkt * g.dh, 0};
    PHK_TRY(sgemm_batched(B.dS, 1, nkt, B.qh, g.dh, 1, preK, g.dh, nkt, g.dh, g.n, 0, bk, st, bf16_products));  // dS^T . qh
    const GemmBatch bv{(int)bh, g.H, (int64_t)g.H * g.n * nkt, (int64_t)g.n * nkt, (int64_t)g.n * I, (int64_t)g.dh,
                       (int64_t)g.H * nkt * g.dh, (int64_t)nkt * g.dh};
    PHK_TRY(sgemm_batched(B.P, 1, nkt, dO, I, 1, preV, g.dh, nkt, g.dh, g.n, 0, bv, st, bf16_products));     // P^T . dO
  }
  PHK_KERNEL_LAUNCH(attn_bwd_dq_kernel, dim3((unsigned)((bh * g.n + 7) / 8)), dim3(256), (size_t)(0), st, q, B.kh, B.dS, A.q_scale, dq, (float*)G.q_scale, (const float*)preQ, g);
  PHK_LAUNCH_CHECK();
  PHK_KERNEL_LAUNCH(attn_bwd_dkv_kernel, dim3((unsigned)((bh * nkt + 7) / 8)), dim3(256), (size_t)(0), st, kv, A.null_kv, B.qh, dO, B.P, B.dS, A.k_scale, dkv,
                                                                     (float*)G.null_kv, (float*)G.k_scale, (const float*)preK, (const float*)preV, g);
  PHK_LAUNCH_CHECK();
  if (dbias) {
    const int64_t total = (int64_t)g.H * g.n * g.m;
    PHK_KERNEL_LAUNCH(attn_bwd_dbias_kernel, dim3((unsigned)((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096)), dim3(256), (size_t)(0), st, B.dS, dbias, g);
    PHK_LAUNCH_CHECK();
  }
  return 0;
}

// Attention forward with dropout on the probabilities (attention.py:177): the explicit path of the backward's
// recomputation -- prep, S = qh.kh^T, softmax + dropout, then O = P_drop.vv written token-major into o [b*n, I].
// fp32 products in both precision modes (the attention core is fp32).  Uses the backward's scratch (qh, kh, vv, P).
int attention_forward_dropout(const float* q, const float* kv, const phk_attn_t& A, const float* bias,
                              const uint8_t* key_mask, float* o, const AttnBwdGeom& g, float* scratch, cudaStream_t st,
                              const DropSite& drop) {
  PHK_REQUIRE(g.dh <= 32 * kDPL, PHK_E_UNSUPPORTED, "train: dim_head > 128");
  PHK_REQUIRE(g.nnull == 0 || A.null_kv, PHK_E_ARG, "train: null_kv missing");
  const int nkt = g.nnull + g.m;
  const int64_t bh = (int64_t)g.b * g.H;
  float* qh = scratch;
  float* kh = qh + bh * g.n * g.dh;
  float* vv = kh + bh * nkt * g.dh;
  float* P = vv + bh * nkt * g.dh;
  const int64_t prep_warps = bh * (g.n + nkt);
  PHK_KERNEL_LAUNCH(attn_bwd_prep_kernel, dim3((unsigned)((prep_warps + 7) / 8)), dim3(256), (size_t)(0), st, q, kv, A.null_kv, A.q_scale, A.k_scale, qh, kh, vv, g);
  PHK_LAUNCH_CHECK();
  const GemmBatch bs{(int)bh, 1, (int64_t)g.n * g.dh, 0, (int64_t)nkt * g.dh, 0, (int64_t)g.n * nkt, 0};
  PHK_TRY(sgemm_batched(qh, g.dh, 1, kh, 1, g.dh, P, nkt, g.n, nkt, g.dh, 0, bs, st));
  PHK_KERNEL_LAUNCH(attn_fwd_softmax_dropout_kernel, dim3((unsigned)((bh * g.n + 7) / 8)), dim3(256), (size_t)(0), st, bias, key_mask, P, g, drop);
  PHK_LAUNCH_CHECK();
  // o[(bi, i), h * dh + d] = sum_j P[bi, h, i, j] vv[bi, h, j, d]
  const int I = g.H * g.dh;
  const GemmBatch bo{(int)bh, g.H, (int64_t)g.H * g.n * nkt, (int64_t)g.n * nkt, (int64_t)g.H * nkt * g.dh,
                     (int64_t)nkt * g.dh, (int64_t)g.n * I, (int64_t)g.dh};
  return sgemm_batched(P, nkt, 1, vv, g.dh, 1, o, I, g.n, g.dh, nkt, 0, bo, st);
}

// ------------------------------------------------------------------------------------------------------------------
// PEG backward (attention.py:64-85 + residual; mirror peg_bwd), layout 0 (rows are the logical (b,t,h,w) order):
//   y[o] = x[o] + b + sum_tap w[tap] * x[o + off(tap)],  off = (kt - pad_t0, kh - 1, kw - 1)
//   dx[p] = dy[p] + sum_tap w[tap] * dy[p - off(tap)] ;  dw[tap] += sum_o dy[o] * x[o + off(tap)] ;  db += sum_o dy[o]
// One CTA per position (neighbour rows resolved once), threads over channels.  The weights arrive tap-major [27, D]
// (the forward's layout); the gradient is accumulated in the parameter's own layout dsconv.weight[D, 1, 3, 3, 3].
// ------------------------------------------------------------------------------------------------------------------
// dw[d, tap] += sum_o dy[o, d] * x[o + off(tap), d]: one CTA per (tap, chunk of positions), the sum over the chunk stays in
// registers (threads over channels, coalesced rows) and leaves as ONE atomic per (channel, tap, chunk) -- the per-position
// atomics this replaces (27 * D per position onto 27 * D addresses) took 0.5 ms per layer at 2304 positions.
constexpr int PEG_DW_CHUNKS = 16, PEG_DW_MAXJ = 8;  // D <= 128 * 8
__global__ void __launch_bounds__(128) peg_bwd_dw_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                         float* __restrict__ dw, int64_t P, int T, int H, int W, int D,
                                                         int pad_t0) {
  const int tap = blockIdx.x;
  const int kt = tap / 9, kh = (tap / 3) % 3, kw = tap % 3;
  const int HW = H * W;
  const int64_t per = (P + gridDim.y - 1) / gridDim.y;
  const int64_t p0 = (int64_t)blockIdx.y * per, p1 = p0 + per < P ? p0 + per : P;
  float acc[PEG_DW_MAXJ];
#pragma unroll
  for (int j = 0; j < PEG_DW_MAXJ; ++j) acc[j] = 0.f;
  for (int64_t p = p0; p < p1; ++p) {
    int rem = (int)(p % ((int64_t)T * HW));
    const int64_t bi = p / ((int64_t)T * HW);
    const int t = rem / HW; rem -= t * HW;
    const int h = rem / W;
    const int wq = rem - h * W;
    const int ts = t + (kt - pad_t0), hs = h + (kh - 1), ws = wq + (kw - 1);
    if (ts < 0 || ts >= T || hs < 0 || hs >= H || ws < 0 || ws >= W) continue;  // uniform over the CTA
    const int64_t src = ((bi * T + ts) * H + hs) * W + ws;
#pragma unroll
    for (int j = 0; j < PEG_DW_MAXJ; ++j) {
      const int d = threadIdx.x + 128 * j;
      if (d < D) acc[j] = fmaf(dy[p * D + d], x[src * D + d], acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < PEG_DW_MAXJ; ++j) {
    const int d = threadIdx.x + 128 * j;
    if (d < D && p1 > p0) atomicAdd(dw + (int64_t)d * 27 + tap, acc[j]);  // dsconv.weight[d, 0, kt, kh, kw]
  }
}

__global__ void __launch_bounds__(128) peg_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                      const float* __restrict__ dy, float* __restrict__ dx,
                                                      int T, int H, int W, int D, int pad_t0) {
  __shared__ int s_out[27];  // output position that reads THIS position through tap, or -1
  const int p = blockIdx.x;
  const int HW = H * W;
  if (threadIdx.x < 27) {
    int rem = p % (T * HW);
    const int bi = p / (T * HW);
    const int t = rem / HW; rem -= t * HW;
    const int h = rem / W;
    const int wq = rem - h * W;
    const int kt = threadIdx.x / 9, kh = (threadIdx.x / 3) % 3, kw = threadIdx.x % 3;
    const int to = t - (kt - pad_t0), ho = h - (kh - 1), wo = wq - (kw - 1);
    s_out[threadIdx.x] = (to >= 0 && to < T && ho >= 0 && ho < H && wo >= 0 && wo < W) ? ((bi * T + to) * H + ho) * W + wo : -1;
  }
  __syncthreads();
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const float dyp = dy[(int64_t)p * D + d];
    float acc = dyp;
#pragma unroll
    for (int tap = 0; tap < 27; ++tap) {
      const int o = s_out[tap];
      if (o >= 0) acc = fmaf(w[(int64_t)tap * D + d], dy[(int64_t)o * D + d], acc);
    }
    dx[(int64_t)p * D + d] = acc;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Embedding backward (phenaki_pytorch.py:194-199): x = tok[id] + pos[p]; the gradient-shrink trick lets only the
// alpha branch carry gradient.  dtok[id] += a * dx ; dpos[p] += a * dx
// ------------------------------------------------------------------------------------------------------------------
__global__ void embed_bwd_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dx, float* __restrict__ dtok,
                                 float* __restrict__ dpos, int n, int dim, float alpha, int vocab_rows) {
  const int64_t row = blockIdx.x;
  int64_t id = ids[row];
  id = id < 0 ? 0 : (id >= vocab_rows ? vocab_rows - 1 : id);  // never scatter outside the table (see token_embed_kernel)
  const int p = (int)(row % n);
  for (int c = threadIdx.x; c < dim; c += blockDim.x) {
    const float v = alpha * dx[row * dim + c];
    atomicAdd(dtok + id * dim + c, v);
    atomicAdd(dpos + (int64_t)p * dim + c, v);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// ContinuousPositionBias backward (attention.py:257-275): bias[h,i,j] = table[u(i,j), h], table = MLP(in[u]).
// The MLP runs over the U distinct coordinate deltas; its backward is three dgrad/wgrad pairs on [U, .] matrices.
// ------------------------------------------------------------------------------------------------------------------
__global__ void cpb_inputs_kernel(float* __restrict__ in, int nd, int d0, int d1, int d2) {
  const int U = (2 * d0 - 1) * (2 * d1 - 1) * (2 * d2 - 1);
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= U) return;
  const int s1 = 2 * d1 - 1, s2 = 2 * d2 - 1;
  const int delta[3] = {u / (s1 * s2) - (d0 - 1), (u / s2) % s1 - (d1 - 1), u % s2 - (d2 - 1)};
  for (int i = 0; i < nd; ++i) {
    const int a = delta[i] < 0 ? -delta[i] : delta[i];
    const float sg = delta[i] > 0 ? 1.f : (delta[i] < 0 ? -1.f : 0.f);
    in[(int64_t)u * nd + i] = sg * logf((float)(a + 1));  // sign(rel) * log(|rel| + 1)  (attention.py:266)
  }
}
// y = leaky_relu(y + bias, 0.1) in place (rows x cols)
__global__ void bias_lrelu_kernel(float* __restrict__ y, const float* __restrict__ bias, int64_t rows, int cols) {
  const int64_t total = rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = y[i] + bias[i % cols];
    y[i] = v > 0.f ? v : 0.1f * v;
  }
}
// d *= (act > 0 ? 1 : 0.1): leaky-relu derivative read off the (sign-preserving) activation
__global__ void lrelu_bwd_kernel(float* __restrict__ d, const float* __restrict__ act, int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    d[i] *= act[i] > 0.f ? 1.0f : 0.1f;
}
// dtable[u(i,j), h] += dbias[h, i, j]
__global__ void cpb_dtable_kernel(const float* __restrict__ dbias, float* __restrict__ dtable, int heads, int d0, int d1,
                                  int d2) {
  const int n = d0 * d1 * d2;
  const int64_t total = (int64_t)n * n;
  const int s1 = 2 * d1 - 1, s2 = 2 * d2 - 1;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / n), j = (int)(idx % n);
    const int i0 = i / (d1 * d2), i1 = (i / d2) % d1, i2 = i % d2;
    const int j0 = j / (d1 * d2), j1 = (j / d2) % d1, j2 = j % d2;
    const int u = ((i0 - j0 + d0 - 1) * s1 + (i1 - j1 + d1 - 1)) * s2 + (i2 - j2 + d2 - 1);
    for (int h = 0; h < heads; ++h) atomicAdd(dtable + (int64_t)u * heads + h, dbias[(int64_t)h * total + idx]);
  }
}

inline unsigned ew_grid(int64_t total) {
  const int64_t b = (total + 255) / 256;
  return (unsigned)(b < 1 ? 1 : (b > kNumSMs * 16 ? kNumSMs * 16 : b));
}

int64_t cpb_bwd_scratch_floats(const phk_cpb_t& c, int d0, int d1, int d2) {
  const int64_t U = (int64_t)(2 * d0 - 1) * (2 * d1 - 1) * (2 * d2 - 1);
  return U * (c.num_dims + 4 * (int64_t)c.hidden + c.heads) + 64;
}

int cpb_backward(const phk_cpb_t& c, const phk_cpb_t& G, const float* dbias, int d0, int d1, int d2, float* scratch,
                 cudaStream_t st) {
  const int64_t U = (int64_t)(2 * d0 - 1) * (2 * d1 - 1) * (2 * d2 - 1);
  const int nd = c.num_dims, hid = c.hidden, H = c.heads;
  float* in = scratch;
  float* a1 = in + U * nd;
  float* a2 = a1 + U * hid;
  float* da1 = a2 + U * hid;
  float* da2 = da1 + U * hid;
  float* dtable = da2 + U * hid;
  PHK_KERNEL_LAUNCH(cpb_inputs_kernel, dim3((unsigned)((U + 127) / 128)), dim3(128), (size_t)(0), st, in, nd, d0, d1, d2);
  PHK_LAUNCH_CHECK();
  // forward activations: a1 = lrelu(in W0^T + b0), a2 = lrelu(a1 W1^T + b1)     (B(k,n) = W[n*K + k])
  PHK_TRY(sgemm(in, nd, 1, c.w0, 1, nd, a1, hid, U, hid, nd, 0, st));
  PHK_KERNEL_LAUNCH(bias_lrelu_kernel, dim3(ew_grid(U * hid)), dim3(256), (size_t)(0), st, a1, c.b0, U, hid);
  PHK_LAUNCH_CHECK();
  PHK_TRY(sgemm(a1, hid, 1, c.w1, 1, hid, a2, hid, U, hid, hid, 0, st));
  PHK_KERNEL_LAUNCH(bias_lrelu_kernel, dim3(ew_grid(U * hid)), dim3(256), (size_t)(0), st, a2, c.b1, U, hid);
  PHK_LAUNCH_CHECK();
  // dtable[u, h] = sum over the (i, j) pairs with delta u
  PHK_CUDA(cudaMemsetAsync(dtable, 0, U * H * sizeof(float), st));
  const int64_t nn = (int64_t)d0 * d1 * d2 * d0 * d1 * d2;
  PHK_KERNEL_LAUNCH(cpb_dtable_kernel, dim3(ew_grid(nn)), dim3(256), (size_t)(0), st, dbias, dtable, H, d0, d1, d2);
  PHK_LAUNCH_CHECK();
  // last layer: table = a2 W2^T + b2
  PHK_TRY(wgrad(dtable, a2, (float*)G.w2, U, H, hid, st));
  PHK_TRY(colsum(dtable, U, H, H, (float*)G.b2, st));
  PHK_TRY(dgrad(dtable, c.w2, da2, U, H, hid, 0, st));
  PHK_KERNEL_LAUNCH(lrelu_bwd_kernel, dim3(ew_grid(U * hid)), dim3(256), (size_t)(0), st, da2, a2, U * hid);
  PHK_LAUNCH_CHECK();
  PHK_TRY(wgrad(da2, a1, (float*)G.w1, U, hid, hid, st));
  PHK_TRY(colsum(da2, U, hid, hid, (float*)G.b1, st));
  PHK_TRY(dgrad(da2, c.w1, da1, U, hid, hid, 0, st));
  PHK_KERNEL_LAUNCH(lrelu_bwd_kernel, dim3(ew_grid(U * hid)), dim3(256), (size_t)(0), st, da1, a1, U * hid);
  PHK_LAUNCH_CHECK();
  PHK_TRY(wgrad(da1, in, (float*)G.w0, U, hid, nd, st));
  PHK_TRY(colsum(da1, U, hid, hid, (float*)G.b0, st));
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// Losses.  MaskGit: mean cross entropy over the masked rows (phenaki_pytorch.py:636-640, F.cross_entropy of
// logits[mask]); dlogits = (softmax - onehot) * scale / n_masked on masked rows, 0 elsewhere (written IN PLACE).
// Critic: mean BCE-with-logits over all rows (:672-675); dscore = (sigmoid - label) * scale / rows.
// row_loss[r] is reduced by loss_reduce_kernel (one CTA: deterministic).
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mask_count_kernel(const uint8_t* __restrict__ mask, int64_t rows,
                                                         float* __restrict__ count) {
  __shared__ float red[32];
  float a = 0.f;
  for (int64_t r = threadIdx.x; r < rows; r += blockDim.x) a += mask[r] ? 1.f : 0.f;
  a = block_sum(a, red);
  if (threadIdx.x == 0) *count = fmaxf(a, 1.f);
}

__global__ void __launch_bounds__(256) ce_rows_kernel(float* __restrict__ logits, const int64_t* __restrict__ targets,
                                                      const uint8_t* __restrict__ mask, const float* __restrict__ count,
                                                      float scale, float* __restrict__ row_loss, int V) {
  __shared__ float red[32];
  __shared__ float bcast;
  const int64_t r = blockIdx.x;
  float* lr = logits + r * (int64_t)V;
  if (!mask[r]) {
    for (int v = threadIdx.x; v < V; v += blockDim.x) lr[v] = 0.f;
    if (threadIdx.x == 0) row_loss[r] = 0.f;
    return;
  }
  float mx = -FLT_MAX;
  for (int v = threadIdx.x; v < V; v += blockDim.x) mx = fmaxf(mx, lr[v]);
  mx = warp_max(mx);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = red[0];
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k) m = fmaxf(m, red[k]);
    bcast = m;
  }
  __syncthreads();
  mx = bcast;
  float s = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) s += expf(lr[v] - mx);
  s = block_sum(s, red);
  const int64_t tgt = targets[r];
  const float lse = mx + logf(s);
  const float tl = lr[tgt];
  __syncthreads();  // every thread has read lr[tgt] before it is overwritten
  const float k = scale / *count;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float p = expf(lr[v] - mx) / s;
    lr[v] = (p - (v == tgt ? 1.f : 0.f)) * k;
  }
  if (threadIdx.x == 0) row_loss[r] = (lse - tl) / *count;
}

// one warp per row: score = emb . w + b ; BCE with logits ; dscore
__global__ void __launch_bounds__(256) bce_rows_kernel(const float* __restrict__ emb, const float* __restrict__ w,
                                                       const float* __restrict__ bias, const float* __restrict__ labels,
                                                       float scale, float* __restrict__ row_loss,
                                                       float* __restrict__ dscore, int64_t rows, int dim) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  float a = 0.f;
  for (int c = lane; c < dim; c += 32) a = fmaf(emb[r * dim + c], w[c], a);
  a = warp_sum(a) + bias[0];
  if (lane == 0) {
    const float y = labels[r];
    row_loss[r] = (fmaxf(a, 0.f) - a * y + log1pf(expf(-fabsf(a)))) / (float)rows;
    dscore[r] = (1.0f / (1.0f + expf(-a)) - y) * scale / (float)rows;
  }
}

__global__ void __launch_bounds__(1024) loss_reduce_kernel(const float* __restrict__ row_loss, int64_t rows,
                                                           float* __restrict__ loss) {
  __shared__ float red[32];
  float a = 0.f;
  for (int64_t r = threadIdx.x; r < rows; r += blockDim.x) a += row_loss[r];
  a = block_sum(a, red);
  if (threadIdx.x == 0) *loss = a;
}

// demb[r, :] = dscore[r] * w
__global__ void outer_kernel(const float* __restrict__ dscore, const float* __restrict__ w, float* __restrict__ out,
                             int64_t rows, int dim) {
  const int64_t total = rows * dim;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = dscore[i / dim] * w[i % dim];
}

struct Arena {
  char* base; int64_t size; int64_t off;
  float* f(int64_t floats) {
    const int64_t o = (off + 255) & ~int64_t(255);
    off = o + floats * 4;
    return (off <= size && base) ? reinterpret_cast<float*>(base + o) : nullptr;
  }
};

struct LayerSave {  // activations of one transformer layer kept for the backward pass (fp32)
  float *x0, *x1, *xn1, *q1, *kv1, *o1, *x2, *ctxn, *ckv, *xn2, *q2, *o2, *x3, *xn3, *h, *g;
};

int64_t layer_save_floats(const phk_transformer_t* T, const phk_layer_t& L, int64_t R, int64_t CR) {
  const int64_t D = T->dim, I = (int64_t)T->heads * T->dim_head;
  int64_t f = R * (D * 6 + I * 4 + 3 * (int64_t)L.ff.inner);  // x0 x1 xn1 x2 x3 xn3 | q1 kv1(2) o1 | h(2) g
  if (L.has_cross) f += CR * (L.cross_attn.dim_context + 2 * I) + R * (D + 2 * I);  // ctxn ckv | xn2 q2 o2
  return f + 64 * 20;
}

// elements of ONE bf16 operand buffer of the tensor-core products (bf16 mode): every operand of every product of the
// step -- activations / gradients [tokens, width] and weights [width, feature], straight or transposed, leading
// dimension padded to 8 -- fits
int64_t tc_scratch_elems(const phk_maskgit_t* m, int64_t R, int64_t CR, bool bce) {
  const phk_transformer_t* T = &m->transformer;
  int64_t inner = 0, dc = 0;
  for (int l = 0; l < T->depth; ++l) {
    if (T->layers[l].ff.inner > inner) inner = T->layers[l].ff.inner;
    if (T->layers[l].has_cross && T->layers[l].cross_attn.dim_context > dc) dc = T->layers[l].cross_attn.dim_context;
  }
  const int64_t I = (int64_t)T->heads * T->dim_head, D = m->dim;
  int64_t width = 2 * inner;
  if (2 * I > width) width = 2 * I;
  if (D > width) width = D;
  if (dc > width) width = dc;
  if (!bce && m->num_tokens > width) width = m->num_tokens;
  int64_t feat = D;
  if (I > feat) feat = I;
  if (inner > feat) feat = inner;
  if (dc > feat) feat = dc;
  const int64_t tokens = pad8(R > CR ? R : CR) + 8;
  return (tokens > feat + 8 ? tokens : feat + 8) * (width + 8);
}

// Counter layout of one step's dropout masks (include/phk.h, phk_dropout_t): per layer, in order, the self-attention
// probabilities [b, H, n, n], the cross-attention probabilities [b, H, n, nnull + L] when the layer runs cross-attention
// (L > 0), the FF hidden [b*n, inner]; each site takes ceil(count / 4) counters right after the previous one.
// bases (optional, [depth][3]): the first counter of each site, relative to the step's offset.  Returns the total.
uint64_t dropout_layout(const phk_maskgit_t* m, int b, int n, int L, uint64_t (*bases)[3]) {
  const phk_transformer_t* T = &m->transformer;
  const uint64_t bh = (uint64_t)b * T->heads;
  uint64_t c = 0;
  for (int l = 0; l < T->depth; ++l) {
    const phk_layer_t& Ly = T->layers[l];
    const uint64_t cross = Ly.has_cross && L > 0 ? bh * n * (uint64_t)(Ly.cross_attn.num_null_kv + L) : 0;
    const uint64_t count[3] = {bh * n * n, cross, (uint64_t)b * n * Ly.ff.inner};
    for (int s = 0; s < 3; ++s) {
      if (bases) bases[l][s] = c;
      c += (count[s] + 3) / 4;
    }
  }
  return c;
}

}  // namespace
}  // namespace phk

using namespace phk;

// Data-parallel overlap (SURVEY 8e): the caller may hand in CUDA events that the NEXT phk_maskgit_train_step call of this
// thread records on its stream as groups of gradients become final -- events[0]: the head + norm_out, events[1 + k]:
// transformer layer depth-1-k (backward order), events[depth + 1]: embeddings + position-bias MLP = everything.  A side
// stream can then all-reduce each finished slice of the flat gradient bucket while the layers below still run.
static thread_local void** g_progress_events = nullptr;
static thread_local int g_progress_count = 0;
extern "C" int phk_train_set_progress_events(void** events, int32_t count) {
  g_progress_events = events;
  g_progress_count = events ? count : 0;
  return 0;
}
static inline int progress_mark(void** ev, int n, int idx, cudaStream_t st) {
  if (ev && idx < n && ev[idx]) PHK_CUDA(cudaEventRecord(reinterpret_cast<cudaEvent_t>(ev[idx]), st));
  return 0;
}

extern "C" int64_t phk_maskgit_train_workspace_bytes(const phk_maskgit_t* m, int32_t b, int32_t n, int32_t L,
                                                     int32_t bce_head, int32_t prec) {
  if (!m || b <= 0 || n <= 0 || L < 0 || !m->transformer.layers) return -1;
  const phk_transformer_t* T = &m->transformer;
  const int64_t R = (int64_t)b * n, CR = (int64_t)b * L, D = m->dim, I = (int64_t)T->heads * T->dim_head;
  int64_t inner = 0, dc = 0, f = 0;
  for (int l = 0; l < T->depth; ++l) {
    f += layer_save_floats(T, T->layers[l], R, CR);
    if (T->layers[l].ff.inner > inner) inner = T->layers[l].ff.inner;
    if (T->layers[l].has_cross && T->layers[l].cross_attn.dim_context > dc) dc = T->layers[l].cross_attn.dim_context;
  }
  f += R * D * 2;                                            // x (embedding output), final embeddings
  f += bce_head ? 3 * R : R * (int64_t)m->num_tokens + 2 * R;  // (d)logits in place or the differentiated copy; row losses
  f += R * (D * 3 + I * 4 + 3 * inner) + CR * (2 * I + dc);  // dxa dxb dtmp | dq dkv(2) do | dh(2) dg | dckv dctxn
  f += 2 * (R > CR ? R : CR);                                // LayerNorm statistics
  const int64_t a1 = attn_bwd_scratch_floats(b, T->heads, n, n, T->dim_head);
  const int64_t a2 = attn_bwd_scratch_floats(b, T->heads, n, L + 8, T->dim_head);
  f += a1 > a2 ? a1 : a2;
  if (m->has_bias) {
    // position bias and its gradient [heads, n, n]; the MLP runs over U = prod(2 d_i - 1) <= 8 n coordinate deltas
    const int64_t U = 8 * (int64_t)n;
    f += 2 * (int64_t)T->heads * n * n + U * m->pos_bias.heads + U * (3 + 4 * (int64_t)m->pos_bias.hidden + m->pos_bias.heads) + 128;
  }
  int64_t bytes = f * 4 + 256 * 64;
  if (prec == PHK_PREC_BF16) bytes += 2 * (tc_scratch_elems(m, R, CR, bce_head != 0) * 2 + 256);
  return bytes;
}

extern "C" int64_t phk_maskgit_train_dropout_counters(const phk_maskgit_t* m, int32_t b, int32_t n, int32_t L) {
  if (!m || b <= 0 || n <= 0 || L < 0 || !m->transformer.layers) return -1;
  return (int64_t)dropout_layout(m, b, n, L, nullptr);
}

// See include/phk.h.  grads: a table of the SAME layout as `m` whose float pointers address zero-filled gradient
// buffers (bf16 members unused); every parameter gradient is accumulated into it.
extern "C" int phk_maskgit_train_step(const phk_maskgit_t* m, const phk_maskgit_t* grads, const int64_t* ids_in,
                                      const int64_t* targets, const uint8_t* token_mask, const float* labels, int32_t b,
                                      int32_t n, int32_t pt, int32_t ph, int32_t pw, const float* context, int32_t L,
                                      const uint8_t* text_mask, const uint8_t* video_mask, float loss_scale,
                                      float* loss_out, float* logits_out, void* workspace, int64_t workspace_bytes,
                                      int32_t prec, phk_stream_t s, const phk_dropout_t* dropout) {
  PHK_REQUIRE(m && grads && ids_in && loss_out && workspace, PHK_E_ARG, "maskgit_train_step: null pointer");
  PHK_REQUIRE(b > 0 && n > 0 && (int64_t)pt * ph * pw == n, PHK_E_SHAPE, "video patch shape must cover the token sequence");
  PHK_REQUIRE(n <= m->max_seq_len, PHK_E_SHAPE,
              "the video token sequence length is greater than max_seq_len (phenaki_pytorch.py:196)");
  // head: labels given -> Linear(dim, 1) + BCE with logits (TokenCritic, or SelfCritic.to_pred on a MaskGit body,
  // phenaki_pytorch.py:307-336); otherwise to_logits + masked cross entropy
  const bool bce = labels != nullptr;
  PHK_REQUIRE(bce || (targets && token_mask), PHK_E_ARG,
              "maskgit_train_step: pass labels (critic head) or targets + token_mask (MaskGit head)");
  PHK_REQUIRE(bce || !m->is_critic, PHK_E_ARG, "maskgit_train_step: a TokenCritic table needs labels");
  PHK_REQUIRE(!(bce && logits_out), PHK_E_ARG, "maskgit_train_step: the critic head has no logits to hand back");
  PHK_REQUIRE(!context || (text_mask && L > 0), PHK_E_ARG, "maskgit_train_step: context without text mask / length");
  PHK_REQUIRE(prec == PHK_PREC_F32 || prec == PHK_PREC_BF16, PHK_E_ARG, "maskgit_train_step: unknown precision mode");
  PHK_REQUIRE(workspace_bytes >= phk_maskgit_train_workspace_bytes(m, b, n, L, bce ? 1 : 0, prec), PHK_E_WORKSPACE,
              "maskgit_train_step: workspace too small");
  const phk_transformer_t* T = &m->transformer;
  const phk_transformer_t* GT = &grads->transformer;
  PHK_REQUIRE(T->layers && GT->layers && T->depth > 0 && GT->depth == T->depth && !T->causal, PHK_E_ARG,
              "maskgit_train_step: transformer table / gradient table mismatch");
  PHK_REQUIRE(m->dim % 4 == 0, PHK_E_UNSUPPORTED, "maskgit_train_step: dim must be a multiple of 4");
  PHK_REQUIRE(!dropout || (dropout->attn_p >= 0.f && dropout->attn_p <= 1.f && dropout->ff_p >= 0.f && dropout->ff_p <= 1.f),
              PHK_E_ARG, "maskgit_train_step: dropout probabilities must lie in [0, 1]");
  const bool drop_on = dropout && (dropout->attn_p > 0.f || dropout->ff_p > 0.f);
  cudaStream_t st = to_stream(s);
  void** prog = g_progress_events;  // one-shot: consumed by this call
  const int nprog = g_progress_count;
  g_progress_events = nullptr; g_progress_count = 0;
  const int D = m->dim, H = T->heads, DH = T->dim_head, I = H * DH, V = m->num_tokens;
  const int64_t R = (int64_t)b * n, CR = (int64_t)b * L;
  Arena ar{(char*)workspace, workspace_bytes, 0};
  TcScratch tc{nullptr, nullptr, 0};
  if (prec == PHK_PREC_BF16) {  // operand buffers of the wgmma products (activations stay fp32 everywhere else)
    tc.elems = tc_scratch_elems(m, R, CR, bce);
    tc.a = reinterpret_cast<__nv_bfloat16*>(ar.f((tc.elems + 1) / 2));
    tc.b = reinterpret_cast<__nv_bfloat16*>(ar.f((tc.elems + 1) / 2));
    PHK_REQUIRE(tc.a && tc.b, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (tensor-core operands)");
  }

  // ---------------------------------------------------------------- forward (saving activations)
  float* x = ar.f(R * D);
  float* emb = ar.f(R * D);
  float* bias = nullptr;
  float* dbias = nullptr;
  if (m->has_bias) {
    bias = ar.f((int64_t)H * n * n);
    dbias = ar.f((int64_t)H * n * n);
    float* sc = ar.f(phk_cpb_scratch_floats(&m->pos_bias, pt, ph, pw));
    PHK_REQUIRE(bias && dbias && sc, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (bias)");
    PHK_TRY(phk_cpb_bias(&m->pos_bias, pt, ph, pw, sc, bias, s));
    PHK_CUDA(cudaMemsetAsync(dbias, 0, (int64_t)H * n * n * 4, st));
  }
  PHK_REQUIRE(x && emb, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small");
  PHK_TRY(phk_token_embed(ids_in, m->token_emb, m->pos_emb, x, b, n, D, m->num_tokens + 1,
                          m->is_critic ? -1.f : m->shrink_alpha, 1, s));
  LayerSave* sv = new (std::nothrow) LayerSave[T->depth];
  PHK_REQUIRE(sv, PHK_E_ARG, "maskgit_train_step: out of host memory");
  struct Free { LayerSave* p; ~Free() { delete[] p; } } free_sv{sv};
  // dropout: site s of layer l (0 self-attention, 1 cross-attention, 2 FF) draws from counters offset + bases[l][s]
  uint64_t (*bases)[3] = drop_on ? new (std::nothrow) uint64_t[T->depth][3] : nullptr;
  PHK_REQUIRE(!drop_on || bases, PHK_E_ARG, "maskgit_train_step: out of host memory");
  struct FreeBases { uint64_t (*p)[3]; ~FreeBases() { delete[] p; } } free_bases{bases};
  if (drop_on) dropout_layout(m, b, n, context ? L : 0, bases);
  auto site = [&](float p, int l, int k) {  // p == 0: the site is off
    DropSite d{0.f, 0.f, 0u, 0u, 0u};
    if (drop_on && p > 0.f) {
      d.p = p; d.scale = 1.0f / (1.0f - p);
      d.k0 = (uint32_t)dropout->seed; d.k1 = (uint32_t)(dropout->seed >> 32);
      d.base = dropout->offset + bases[l][k];
    }
    return d;
  };
  const float attn_p = dropout ? dropout->attn_p : 0.f, ff_p = dropout ? dropout->ff_p : 0.f;
  // the attention backward's scratch; the forward's explicit attention path (dropout) uses it too
  const int nk_cross = L + 8;
  const int64_t as1 = attn_bwd_scratch_floats(b, H, n, n, DH), as2 = attn_bwd_scratch_floats(b, H, n, nk_cross, DH);
  float* asc = ar.f(as1 > as2 ? as1 : as2);
  PHK_REQUIRE(asc, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (attention scratch)");
  phk_attn_geom_t ag;
  const float* xin = x;
  for (int l = 0; l < T->depth; ++l) {
    const phk_layer_t& Ly = T->layers[l];
    LayerSave& S = sv[l];
    std::memset(&S, 0, sizeof(S));
    const int inner = Ly.ff.inner;
    PHK_REQUIRE(Ly.has_peg, PHK_E_UNSUPPORTED, "maskgit_train_step: layers without PEG are not supported");
    S.x0 = const_cast<float*>(xin);
    S.x1 = ar.f(R * D); S.xn1 = ar.f(R * D); S.q1 = ar.f(R * I); S.kv1 = ar.f(R * 2 * I); S.o1 = ar.f(R * I);
    S.x2 = ar.f(R * D); S.x3 = ar.f(R * D); S.xn3 = ar.f(R * D); S.h = ar.f(R * 2 * (int64_t)inner); S.g = ar.f(R * (int64_t)inner);
    float* xout = ar.f(R * D);
    PHK_REQUIRE(S.x1 && S.xn1 && S.q1 && S.kv1 && S.o1 && S.x2 && S.x3 && S.xn3 && S.h && S.g && xout, PHK_E_WORKSPACE,
                "maskgit_train_step: workspace too small (activations)");
    // x1 = peg(x0) + x0
    PHK_TRY(phk_peg3d(S.x0, Ly.peg.w, Ly.peg.b, S.x1, b, pt, ph, pw, D, Ly.peg.causal, 0, s));
    // self attention: q from LN(x1), k/v from RAW x1 (attention.py:140-144)
    const phk_attn_t& A = Ly.self_attn;
    PHK_TRY(phk_layernorm(S.x1, A.norm_g, A.norm_b, S.xn1, nullptr, R, D, 0, 0, 0, 0, s));
    PHK_TRY(linear_fwd(prec, tc, S.xn1, A.wq, S.q1, R, I, D, nullptr, nullptr, s));
    PHK_TRY(linear_fwd(prec, tc, S.x1, A.wkv, S.kv1, R, 2 * I, D, nullptr, nullptr, s));
    std::memset(&ag, 0, sizeof(ag));
    ag.n_outer = b; ag.n_inner = 1; ag.n_q = n; ag.n_k = n; ag.heads = H; ag.dim_head = DH; ag.num_null_kv = A.num_null_kv;
    ag.q_outer = (int64_t)n * I; ag.q_tok = I; ag.k_outer = (int64_t)n * 2 * I; ag.k_tok = 2 * I;
    ag.o_outer = ag.q_outer; ag.o_tok = I; ag.mask_off_from = -1; ag.scale = 8.f;
    PHK_REQUIRE(A.num_null_kv == 0, PHK_E_UNSUPPORTED, "maskgit_train_step: self-attention null-kv is not supported");
    const DropSite d_self = site(attn_p, l, 0);
    if (d_self.p > 0.f) {
      const AttnBwdGeom g1{b, H, n, n, 0, DH};
      PHK_TRY(attention_forward_dropout(S.q1, S.kv1, A, bias, video_mask, S.o1, g1, asc, st, d_self));
    } else {
      PHK_TRY(phk_attention(S.q1, S.kv1, A.null_kv, A.q_scale, A.k_scale, bias, video_mask, nullptr, S.o1, &ag, s));
    }
    PHK_TRY(linear_fwd(prec, tc, S.o1, A.wo, S.x2, R, D, I, nullptr, S.x1, s));  // x2 = x1 + o Wo^T
    const bool cross = Ly.has_cross && context;
    if (cross) {
      const phk_attn_t& Cx = Ly.cross_attn;
      const int dc = Cx.dim_context;
      S.ctxn = ar.f(CR * dc); S.ckv = ar.f(CR * 2 * I); S.xn2 = ar.f(R * D); S.q2 = ar.f(R * I); S.o2 = ar.f(R * I);
      PHK_REQUIRE(S.ctxn && S.ckv && S.xn2 && S.q2 && S.o2, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (cross)");
      PHK_TRY(phk_layernorm(context, Cx.ctx_g, Cx.ctx_b, S.ctxn, nullptr, CR, dc, 0, 0, 0, 0, s));
      PHK_TRY(linear_fwd(prec, tc, S.ctxn, Cx.wkv, S.ckv, CR, 2 * I, dc, nullptr, nullptr, s));
      PHK_TRY(phk_layernorm(S.x2, Cx.norm_g, Cx.norm_b, S.xn2, nullptr, R, D, 0, 0, 0, 0, s));
      PHK_TRY(linear_fwd(prec, tc, S.xn2, Cx.wq, S.q2, R, I, D, nullptr, nullptr, s));
      std::memset(&ag, 0, sizeof(ag));
      ag.n_outer = b; ag.n_inner = 1; ag.n_q = n; ag.n_k = L; ag.heads = H; ag.dim_head = DH; ag.num_null_kv = Cx.num_null_kv;
      ag.q_outer = (int64_t)n * I; ag.q_tok = I; ag.k_outer = (int64_t)L * 2 * I; ag.k_tok = 2 * I;
      ag.o_outer = ag.q_outer; ag.o_tok = I; ag.kv_outer_mod = b; ag.mask_outer_mod = b; ag.mask_off_from = -1; ag.scale = 8.f;
      const DropSite d_cross = site(attn_p, l, 1);
      if (d_cross.p > 0.f) {
        PHK_REQUIRE(Cx.num_null_kv <= 8, PHK_E_UNSUPPORTED, "maskgit_train_step: more than 8 null key/values");
        const AttnBwdGeom g2{b, H, n, L, Cx.num_null_kv, DH};
        PHK_TRY(attention_forward_dropout(S.q2, S.ckv, Cx, nullptr, text_mask, S.o2, g2, asc, st, d_cross));
      } else {
        PHK_TRY(phk_attention(S.q2, S.ckv, Cx.null_kv, Cx.q_scale, Cx.k_scale, nullptr, text_mask, nullptr, S.o2, &ag, s));
      }
      PHK_TRY(linear_fwd(prec, tc, S.o2, Cx.wo, S.x3, R, D, I, nullptr, S.x2, s));  // x3 = x2 + o2 Wo^T
    } else {
      PHK_CUDA(cudaMemcpyAsync(S.x3, S.x2, R * D * 4, cudaMemcpyDeviceToDevice, st));
    }
    // feed forward (attention.py:45-53)
    PHK_TRY(phk_layernorm(S.x3, Ly.ff.ln_g, Ly.ff.ln_b, S.xn3, nullptr, R, D, 0, 0, 0, 0, s));
    PHK_TRY(linear_fwd(prec, tc, S.xn3, Ly.ff.w1, S.h, R, 2 * inner, D, nullptr, nullptr, s));
    const DropSite d_ff = site(ff_p, l, 2);
    if (d_ff.p > 0.f) {
      PHK_KERNEL_LAUNCH(geglu_dropout_kernel, dim3(ew_grid_fwd(R * inner)), dim3(256), (size_t)(0), st, S.h, S.g, R, inner, d_ff);
      PHK_LAUNCH_CHECK();
    } else {
      PHK_TRY(phk_geglu(S.h, S.g, R, inner, s));
    }
    PHK_TRY(linear_fwd(prec, tc, S.g, Ly.ff.w2, xout, R, D, inner, nullptr, S.x3, s));  // x4 = x3 + g W2^T
    xin = xout;
  }
  const float* xf = xin;
  PHK_TRY(phk_layernorm(xf, T->out_g, T->out_b, emb, nullptr, R, D, 0, 0, 0, 0, s));

  // ---------------------------------------------------------------- head + loss -> demb
  float* dxa = ar.f(R * D);
  float* dxb = ar.f(R * D);
  float* dtmp = ar.f(R * D);
  float* row_loss = ar.f(R);
  float* cnt = ar.f(64);
  float2* stats = reinterpret_cast<float2*>(ar.f(2 * (R > CR ? R : CR)));
  PHK_REQUIRE(dxa && dxb && dtmp && row_loss && cnt && stats, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (bwd)");
  if (bce) {
    float* dscore = ar.f(R);
    PHK_REQUIRE(dscore, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small");
    PHK_KERNEL_LAUNCH(bce_rows_kernel, dim3((unsigned)((R + 7) / 8)), dim3(256), (size_t)(0), st, emb, m->head_w, m->head_b, labels, loss_scale, row_loss, dscore, R, D);
    PHK_LAUNCH_CHECK();
    PHK_TRY(wgrad(dscore, emb, (float*)grads->head_w, R, 1, D, st));  // [1, dim]: not worth a tensor-core launch
    PHK_TRY(colsum(dscore, R, 1, 1, (float*)grads->head_b, st));
    PHK_KERNEL_LAUNCH(outer_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, dscore, m->head_w, dtmp, R, D);
    PHK_LAUNCH_CHECK();
  } else {
    float* logits = logits_out ? logits_out : ar.f(R * (int64_t)V);
    PHK_REQUIRE(logits, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (logits)");
    PHK_TRY(linear_fwd(prec, tc, emb, m->head_w, logits, R, V, D, m->head_b, nullptr, s));
    float* dl = logits;
    if (logits_out) {  // the caller keeps the logits (critic sampling, :646): differentiate a copy
      dl = ar.f(R * (int64_t)V);
      PHK_REQUIRE(dl, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (dlogits)");
      PHK_CUDA(cudaMemcpyAsync(dl, logits, R * (int64_t)V * 4, cudaMemcpyDeviceToDevice, st));
    }
    PHK_KERNEL_LAUNCH(mask_count_kernel, dim3(1), dim3(256), (size_t)(0), st, token_mask, R, cnt);
    PHK_LAUNCH_CHECK();
    PHK_KERNEL_LAUNCH(ce_rows_kernel, dim3((unsigned)R), dim3(256), (size_t)(0), st, dl, targets, token_mask, cnt, loss_scale, row_loss, V);
    PHK_LAUNCH_CHECK();
    PHK_TRY(wgrad_p(prec, tc, dl, emb, (float*)grads->head_w, R, V, D, s));
    PHK_TRY(colsum(dl, R, V, V, (float*)grads->head_b, st));
    PHK_TRY(dgrad_p(prec, tc, dl, m->head_w, dtmp, R, V, D, 0, s));
  }
  PHK_KERNEL_LAUNCH(loss_reduce_kernel, dim3(1), dim3(1024), (size_t)(0), st, row_loss, R, loss_out);
  PHK_LAUNCH_CHECK();

  // ---------------------------------------------------------------- backward through the transformer
  int64_t inner_max = 0, dc_max = 0;
  for (int l = 0; l < T->depth; ++l) {
    if (T->layers[l].ff.inner > inner_max) inner_max = T->layers[l].ff.inner;
    if (T->layers[l].has_cross && T->layers[l].cross_attn.dim_context > dc_max) dc_max = T->layers[l].cross_attn.dim_context;
  }
  float* dq = ar.f(R * I);
  float* dkv = ar.f(R * 2 * I);
  float* dob = ar.f(R * I);
  float* dh = ar.f(R * 2 * inner_max);
  float* dg = ar.f(R * inner_max);
  float* dckv = context ? ar.f(CR * 2 * I) : nullptr;
  float* dctxn = context ? ar.f(CR * (dc_max > 0 ? dc_max : 1)) : nullptr;
  PHK_REQUIRE(dq && dkv && dob && dh && dg && (!context || (dckv && dctxn)), PHK_E_WORKSPACE,
              "maskgit_train_step: workspace too small (gradients)");
  float* dx = dxa;      // d loss / d (current residual stream)
  float* dx_alt = dxb;
  PHK_TRY(ln_backward(xf, T->out_g, dtmp, dx, 0, (float*)GT->out_g, nullptr, stats, R, D, st));
  PHK_TRY(progress_mark(prog, nprog, 0, st));  // head + norm_out gradients final
  for (int l = T->depth - 1; l >= 0; --l) {
    const phk_layer_t& Ly = T->layers[l];
    const phk_layer_t& Gy = GT->layers[l];
    const LayerSave& S = sv[l];
    const int inner = Ly.ff.inner;
    // feed forward: x4 = x3 + geglu(LN(x3) W1^T) W2^T
    PHK_TRY(dgrad_p(prec, tc, dx, Ly.ff.w2, dg, R, D, inner, 0, s));
    PHK_TRY(wgrad_p(prec, tc, dx, S.g, (float*)Gy.ff.w2, R, D, inner, s));
    PHK_KERNEL_LAUNCH(geglu_bwd_kernel, dim3(ew_grid(R * inner)), dim3(256), (size_t)(0), st, S.h, dg, dh, R, inner, site(ff_p, l, 2));
    PHK_LAUNCH_CHECK();
    PHK_TRY(wgrad_p(prec, tc, dh, S.xn3, (float*)Gy.ff.w1, R, 2 * inner, D, s));
    PHK_TRY(dgrad_p(prec, tc, dh, Ly.ff.w1, dtmp, R, 2 * inner, D, 0, s));
    PHK_TRY(ln_backward(S.x3, Ly.ff.ln_g, dtmp, dx, 1, (float*)Gy.ff.ln_g, (float*)Gy.ff.ln_b, stats, R, D, st));
    // cross attention: x3 = x2 + attn(LN(x2) Wq^T, LN_ctx(context) Wkv^T) Wo^T
    if (S.o2) {
      const phk_attn_t& Cx = Ly.cross_attn;
      const phk_attn_t& Gx = Gy.cross_attn;
      const int dc = Cx.dim_context;
      PHK_REQUIRE(Cx.num_null_kv <= 8, PHK_E_UNSUPPORTED, "maskgit_train_step: more than 8 null key/values");
      PHK_TRY(dgrad_p(prec, tc, dx, Cx.wo, dob, R, D, I, 0, s));
      PHK_TRY(wgrad_p(prec, tc, dx, S.o2, (float*)Gx.wo, R, D, I, s));
      const AttnBwdGeom g2{b, H, n, L, Cx.num_null_kv, DH};
      PHK_TRY(attention_backward(S.q2, S.ckv, Cx, Gx, nullptr, text_mask, dob, dq, dckv, nullptr, g2, asc, st, prec == PHK_PREC_BF16,
                                 site(attn_p, l, 1)));
      PHK_TRY(wgrad_p(prec, tc, dq, S.xn2, (float*)Gx.wq, R, I, D, s));
      PHK_TRY(dgrad_p(prec, tc, dq, Cx.wq, dtmp, R, I, D, 0, s));
      PHK_TRY(ln_backward(S.x2, Cx.norm_g, dtmp, dx, 1, (float*)Gx.norm_g, nullptr, stats, R, D, st));
      PHK_TRY(wgrad_p(prec, tc, dckv, S.ctxn, (float*)Gx.wkv, CR, 2 * I, dc, s));
      PHK_TRY(dgrad_p(prec, tc, dckv, Cx.wkv, dctxn, CR, 2 * I, dc, 0, s));
      PHK_TRY(ln_backward(context, Cx.ctx_g, dctxn, nullptr, 0, (float*)Gx.ctx_g, nullptr, stats, CR, dc, st));
    }
    // self attention: x2 = x1 + attn(LN(x1) Wq^T, x1 Wkv^T) Wo^T
    {
      const phk_attn_t& A = Ly.self_attn;
      const phk_attn_t& GA = Gy.self_attn;
      PHK_TRY(dgrad_p(prec, tc, dx, A.wo, dob, R, D, I, 0, s));
      PHK_TRY(wgrad_p(prec, tc, dx, S.o1, (float*)GA.wo, R, D, I, s));
      const AttnBwdGeom g1{b, H, n, n, 0, DH};
      PHK_TRY(attention_backward(S.q1, S.kv1, A, GA, bias, video_mask, dob, dq, dkv, dbias, g1, asc, st, prec == PHK_PREC_BF16,
                                 site(attn_p, l, 0)));
      PHK_TRY(wgrad_p(prec, tc, dq, S.xn1, (float*)GA.wq, R, I, D, s));
      PHK_TRY(wgrad_p(prec, tc, dkv, S.x1, (float*)GA.wkv, R, 2 * I, D, s));
      PHK_TRY(dgrad_p(prec, tc, dq, A.wq, dtmp, R, I, D, 0, s));
      PHK_TRY(ln_backward(S.x1, A.norm_g, dtmp, dx, 1, (float*)GA.norm_g, nullptr, stats, R, D, st));
      PHK_TRY(dgrad_p(prec, tc, dkv, A.wkv, dx, R, 2 * I, D, 1, s));  // the raw-x path of k, v
    }
    // PEG: x1 = x0 + conv(x0) + b
    PHK_TRY(colsum(dx, R, D, D, (float*)Gy.peg.b, st));
    PHK_REQUIRE(D <= 128 * PEG_DW_MAXJ, PHK_E_UNSUPPORTED, "maskgit_train_step: dim > 1024");
    PHK_KERNEL_LAUNCH(peg_bwd_dw_kernel, dim3(27, PEG_DW_CHUNKS), dim3(128), (size_t)(0), st, S.x0, dx, (float*)Gy.peg.w, R, pt, ph, pw, D, Ly.peg.causal ? 2 : 1);
    PHK_LAUNCH_CHECK();
    PHK_KERNEL_LAUNCH(peg_bwd_kernel, dim3((unsigned)R), dim3(128), (size_t)(0), st, S.x0, Ly.peg.w, dx, dx_alt, pt, ph, pw, D, Ly.peg.causal ? 2 : 1);
    PHK_LAUNCH_CHECK();
    float* t = dx; dx = dx_alt; dx_alt = t;
    // this layer's parameter gradients are final -- except, with a context, the cross-attention's context_norm / to_kv
    // share nothing with other layers either; the position-bias gradient (dbias, all layers) is finished below
    PHK_TRY(progress_mark(prog, nprog, 1 + (T->depth - 1 - l), st));
  }
  // ---------------------------------------------------------------- embeddings, position-bias MLP
  PHK_KERNEL_LAUNCH(embed_bwd_kernel, dim3((unsigned)R), dim3(128), (size_t)(0), st, ids_in, dx, (float*)grads->token_emb, (float*)grads->pos_emb, n, D,
                                               m->is_critic ? 1.0f : m->shrink_alpha, m->num_tokens + 1);
  PHK_LAUNCH_CHECK();
  if (m->has_bias) {
    float* csc = ar.f(cpb_bwd_scratch_floats(m->pos_bias, pt, ph, pw));
    PHK_REQUIRE(csc, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (position-bias backward)");
    PHK_TRY(cpb_backward(m->pos_bias, grads->pos_bias, dbias, pt, ph, pw, csc, st));
  }
  PHK_TRY(progress_mark(prog, nprog, T->depth + 1, st));
  return 0;
}
