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
// by tests/test_gpu_train.py.  The same layer code differentiates the C-ViViT decoder (phk_cvivit_decode_backward) and the
// tokenizer's reconstruction loss through decoder, LFQ and encoder (phk_cvivit_backward), at the end of this file.
#include "phk_common.cuh"
// the kernels of this file are ordinary stream-ordered launches (they do not use programmatic dependent launch)
#define PHK_KERNEL_LAUNCH(kernel, grid, block, smem, st, ...) PHK_CUDA(launch_plain(kernel, grid, block, smem, st, __VA_ARGS__))
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>

namespace phk {
namespace {

constexpr float kLnEps = 1e-5f;
constexpr float kL2Eps = 1e-12f;

// ------------------------------------------------------------------------------------------------------------------
// Deterministic mode (include/phk.h, phk_train_set_deterministic; DESIGN.md section 7.6).  Every reduction that the
// default path finishes with float atomics -- split-K wgrad, bias column sums, LayerNorm gamma / beta, q_scale / k_scale,
// null_kv, the PEG weights, the embeddings and the position-bias table -- then writes per-CTA partial sums to fixed slots
// of a scratch region and adds the slots into the gradient in slot order, or gathers its terms in index order.  Every
// summation order is a function of the call's shapes (and, for the token embedding, of the ids) alone.
// The entry point carves the region from the call's workspace and publishes it in t_det for the duration of the call;
// t_det.p == NULL is the default path.  The reductions run one after another on the call's stream, so each one uses
// the region from its start.
// ------------------------------------------------------------------------------------------------------------------
thread_local int32_t t_det_mode = 0;             // phk_train_set_deterministic: read by the backward entry points
struct DetScratch { float* p; int64_t floats; };
thread_local DetScratch t_det{nullptr, 0};        // the current call's region (NULL: default path)

// Clears t_det when the entry point that published it returns, whichever way it returns.
struct DetScope {
  DetScope() = default;
  DetScope(const DetScope&) = delete;
  ~DetScope() { t_det = DetScratch{nullptr, 0}; }
};

constexpr int kDetRows = 256;  // rows per partial sum of colsum_fixed
inline int64_t det_blocks(int64_t rows) { return (rows + kDetRows - 1) / kDetRows; }

// Fixed-order column sums of x [rows, cols] (leading dimension ld).  CTA (cx, gy) takes 32 columns of the rows
// [gy * per, (gy + 1) * per): warp w adds rows w, w + 8, ... in order, then the 8 warps are added in order.
// to_out == 0: the sum is written to out[gy * cols + c]; to_out == 1: it is added to out[c] (gridDim.y == 1).
__global__ void __launch_bounds__(256) colsum_fixed_kernel(const float* __restrict__ x, int64_t rows, int64_t cols,
                                                           int64_t ld, int64_t per, float* __restrict__ out, int to_out) {
  __shared__ float red[8][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t c = (int64_t)blockIdx.x * 32 + lane;
  const int64_t r0 = (int64_t)blockIdx.y * per, r1 = r0 + per < rows ? r0 + per : rows;
  float a = 0.f;
  if (c < cols)
    for (int64_t r = r0 + w; r < r1; r += 8) a += x[r * ld + c];
  red[w][lane] = a;
  __syncthreads();
  if (w == 0 && c < cols) {
    float s = red[0][lane];
    for (int k = 1; k < 8; ++k) s += red[k][lane];
    if (to_out) out[c] += s;
    else out[(int64_t)blockIdx.y * cols + c] = s;
  }
}
// out[c] += sum_r slots[r, c] for a [nslots, cols] block of partial sums, in one fixed order
int add_slots(const float* slots, int64_t nslots, int64_t cols, float* out, cudaStream_t st) {
  PHK_KERNEL_LAUNCH(colsum_fixed_kernel, dim3((unsigned)((cols + 31) / 32), 1), dim3(256), (size_t)(0), st, slots, nslots, cols, cols, nslots, out, 1);
  PHK_LAUNCH_CHECK();
  return 0;
}
// Floats of scratch colsum_fixed uses for `rows` rows of `cols` columns
inline int64_t colsum_fixed_floats(int64_t rows, int64_t cols) { return det_blocks(rows) * cols; }
// out[c] += sum_r x[r, c] in a fixed order: partial sums of kDetRows-row blocks into `scratch` (cap floats), then
// those partials in block order
int colsum_fixed(const float* x, int64_t rows, int64_t cols, int64_t ld, float* out, float* scratch, int64_t cap,
                 cudaStream_t st) {
  const int64_t G = det_blocks(rows);
  PHK_REQUIRE(scratch && G * cols <= cap, PHK_E_WORKSPACE, "train: deterministic reduction scratch too small");
  PHK_REQUIRE(G <= 65535 && (cols + 31) / 32 < (1LL << 31), PHK_E_UNSUPPORTED, "train: column sum too large");
  PHK_KERNEL_LAUNCH(colsum_fixed_kernel, dim3((unsigned)((cols + 31) / 32), (unsigned)G), dim3(256), (size_t)(0), st, x, rows, cols, ld, (int64_t)kDetRows, scratch, 0);
  PHK_LAUNCH_CHECK();
  return add_slots(scratch, G, cols, out, st);
}

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
    if (t_det.p) {  // deterministic mode: slice z writes its [N, K] product to slot z, the slots are added in order
      PHK_REQUIRE(parts * N * K <= t_det.floats, PHK_E_WORKSPACE, "train: deterministic reduction scratch too small");
      const GemmBatch gb{parts, 1, chunk * N, 0, chunk * K, 0, N * K, 0, (int)M};
      PHK_TRY(sgemm_batched(dY, 1, N, X, K, 1, t_det.p, K, N, K, chunk, 0, gb, st));
      return add_slots(t_det.p, parts, N * K, dW, st);
    }
    const GemmBatch gb{parts, 1, chunk * N, 0, chunk * K, 0, 0, 0, (int)M};
    return sgemm_batched(dY, 1, N, X, K, 1, dW, K, N, K, chunk, 2, gb, st);
  }
  return sgemm(dY, 1, N, X, K, 1, dW, K, N, K, M, 1, st);
}
// Deterministic-mode scratch of wgrad: the split-K slots (0 when the product is not split)
int64_t wgrad_det_floats(int64_t M, int64_t N, int64_t K) {
  return (N * K <= 4 * GB * GB && M >= 1024) ? (M + 255) / 256 * N * K : 0;
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
  if (t_det.p) return colsum_fixed(x, rows, cols, ld, out, t_det.p, t_det.floats, st);
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

// src [rows, cols] (transpose: its transpose) as bf16 with the leading dimension padded to 8 elements
int cast_check(int64_t rows, int64_t cols, bool transpose, int64_t cap, int64_t* ld) {
  PHK_REQUIRE(rows > 0 && cols > 0 && cols < (1LL << 31), PHK_E_ARG, "train: bad operand shape");
  *ld = pad8(transpose ? rows : cols);
  PHK_REQUIRE((transpose ? cols : rows) * *ld <= cap, PHK_E_WORKSPACE, "train: tensor-core operand scratch too small");
  PHK_REQUIRE(!transpose || (rows + 31) / 32 <= 65535, PHK_E_UNSUPPORTED, "train: operand too tall for the transposing cast");
  return 0;
}
int cast_to(const float* src, int64_t rows, int64_t cols, bool transpose, __nv_bfloat16* dst, int64_t ld, cudaStream_t st) {
  if (!transpose) {
    PHK_KERNEL_LAUNCH(cast_bf16_kernel, dim3(ew_grid_fwd(rows * cols)), dim3(256), (size_t)(0), st, src, rows, (int)cols, dst, ld);
  } else {
    PHK_KERNEL_LAUNCH(cast_transpose_bf16_kernel, dim3((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32)), dim3(256), (size_t)(0), st, src, rows, (int)cols, dst, ld);
  }
  PHK_LAUNCH_CHECK();
  return 0;
}
// both operands of one product into tc.a / tc.b: both are checked before either cast launches, so that a refused call
// leaves no work behind
int cast_operands(const TcScratch& tc, const float* a, int64_t ar, int64_t ac, bool at, int64_t* lda, const float* b,
                  int64_t br, int64_t bc, bool bt, int64_t* ldb, cudaStream_t st) {
  PHK_TRY(cast_check(ar, ac, at, tc.elems, lda));
  PHK_TRY(cast_check(br, bc, bt, tc.elems, ldb));
  PHK_TRY(cast_to(a, ar, ac, at, tc.a, *lda, st));
  return cast_to(b, br, bc, bt, tc.b, *ldb, st);
}

// Y[M,N] = X[M,K].W[N,K]^T (+bias) (+residual: `residual` must be Y itself, i.e. Y already holds the residual)
int linear_fwd(int prec, const TcScratch& tc, const float* X, const float* W, float* Y, int64_t M, int64_t N, int64_t K,
               const float* bias, const float* residual, phk_stream_t s) {
  if (prec != PHK_PREC_BF16)
    return phk_gemm_f32(X, K, W, K, Y, N, M, (int32_t)N, (int32_t)K, bias, residual, 0, 0, 0, s);
  int64_t lda = 0, ldw = 0;
  PHK_TRY(cast_operands(tc, X, M, K, false, &lda, W, N, K, false, &ldw, to_stream(s)));
  if (residual && residual != Y) PHK_CUDA(cudaMemcpyAsync(Y, residual, M * N * 4, cudaMemcpyDeviceToDevice, to_stream(s)));
  return phk_gemm_bf16(tc.a, lda, tc.b, ldw, Y, N, M, (int32_t)N, (int32_t)K, bias, residual ? Y : nullptr, 0, 0, 0, 0, s);
}
// dX[M,K] (+)= dY[M,N] . W[N,K]
int dgrad_p(int prec, const TcScratch& tc, const float* dY, const float* W, float* dX, int64_t M, int64_t N, int64_t K,
            int accumulate, phk_stream_t s) {
  if (prec != PHK_PREC_BF16) return dgrad(dY, W, dX, M, N, K, accumulate, to_stream(s));
  int64_t lda = 0, ldw = 0;
  PHK_TRY(cast_operands(tc, dY, M, N, false, &lda, W, N, K, true, &ldw, to_stream(s)));  // dY [M, N], W^T [K, N]
  return phk_gemm_bf16(tc.a, lda, tc.b, ldw, dX, K, M, (int32_t)K, (int32_t)N, nullptr, accumulate ? dX : nullptr, 0, 0, 0, 0, s);
}
// dW[N,K] += dY[M,N]^T . X[M,K]
int wgrad_p(int prec, const TcScratch& tc, const float* dY, const float* X, float* dW, int64_t M, int64_t N, int64_t K,
            phk_stream_t s) {
  if (prec != PHK_PREC_BF16) return wgrad(dY, X, dW, M, N, K, to_stream(s));
  int64_t lda = 0, ldw = 0;
  PHK_TRY(cast_operands(tc, dY, M, N, true, &lda, X, M, K, true, &ldw, to_stream(s)));  // dY^T [N, M], X^T [K, M]
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

// Deterministic mode: the column kernel's sums over kDetRows-row blocks, in colsum_fixed_kernel's order, into
// part_g / part_b [gridDim.y, dim]
__global__ void __launch_bounds__(256) ln_bwd_dgb_fixed_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                               const float2* __restrict__ stats, int64_t rows, int dim,
                                                               float* __restrict__ part_g, float* __restrict__ part_b) {
  __shared__ float rg[8][33], rb[8][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const int64_t r0 = (int64_t)blockIdx.y * kDetRows, r1 = r0 + kDetRows < rows ? r0 + kDetRows : rows;
  float ag = 0.f, ab = 0.f;
  if (c < dim)
    for (int64_t r = r0 + w; r < r1; r += 8) {
      const float2 s = stats[r];
      const float d = dy[r * dim + c];
      ag += d * (x[r * dim + c] - s.x) * s.y;
      ab += d;
    }
  rg[w][lane] = ag;
  rb[w][lane] = ab;
  __syncthreads();
  if (w == 0 && c < dim) {
    float sg = rg[0][lane], sb = rb[0][lane];
    for (int k = 1; k < 8; ++k) { sg += rg[k][lane]; sb += rb[k][lane]; }
    part_g[(int64_t)blockIdx.y * dim + c] = sg;
    if (part_b) part_b[(int64_t)blockIdx.y * dim + c] = sb;
  }
}
inline int64_t ln_det_floats(int64_t rows, int64_t dim) { return 2 * det_blocks(rows) * dim; }

// dx (+)= LN_bwd(x; g)(dy); dgamma += ..; dbeta += .. (dbeta NULL: the custom LayerNorm's beta is a buffer)
int ln_backward(const float* x, const float* g, const float* dy, float* dx, int accumulate, float* dgamma, float* dbeta,
                float2* stats, int64_t rows, int dim, cudaStream_t st) {
  PHK_KERNEL_LAUNCH(ln_bwd_dx_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), (size_t)(0), st, x, g, dy, dx, stats, rows, dim, accumulate);
  PHK_LAUNCH_CHECK();
  if (t_det.p) {
    const int64_t G = det_blocks(rows);
    PHK_REQUIRE(ln_det_floats(rows, dim) <= t_det.floats, PHK_E_WORKSPACE, "train: deterministic reduction scratch too small");
    PHK_REQUIRE(G <= 65535, PHK_E_UNSUPPORTED, "train: LayerNorm backward too tall");
    float* pg = t_det.p;
    float* pb = dbeta ? t_det.p + G * dim : nullptr;
    PHK_KERNEL_LAUNCH(ln_bwd_dgb_fixed_kernel, dim3((unsigned)((dim + 31) / 32), (unsigned)G), dim3(256), (size_t)(0), st, x, dy, (const float2*)stats, rows, dim, pg, pb);
    PHK_LAUNCH_CHECK();
    PHK_TRY(add_slots(pg, G, dim, dgamma, st));
    return dbeta ? add_slots(pb, G, dim, dbeta, st) : 0;
  }
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
// scale_part (deterministic mode, else NULL): the CTA's q_scale sum goes to its slot blockIdx.x instead of dq_scale
__device__ __forceinline__ void attn_bwd_dq_body(const float* __restrict__ q, const float* __restrict__ kh,
                                                 const float* __restrict__ dS, const float* __restrict__ q_scale,
                                                 float* __restrict__ dq, float* __restrict__ dq_scale,
                                                 const float* __restrict__ pre, float* __restrict__ scale_part,
                                                 const AttnBwdGeom& g) {
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
    if (scale_part) scale_part[(int64_t)blockIdx.x * g.dh + threadIdx.x] = a;
    else atomicAdd(dq_scale + threadIdx.x, a);
  }
}
__global__ void __launch_bounds__(256) attn_bwd_dq_kernel(const float* __restrict__ q, const float* __restrict__ kh,
                                                          const float* __restrict__ dS, const float* __restrict__ q_scale,
                                                          float* __restrict__ dq, float* __restrict__ dq_scale,
                                                          const float* __restrict__ pre, AttnBwdGeom g) {
  attn_bwd_dq_body(q, kh, dS, q_scale, dq, dq_scale, pre, nullptr, g);
}
__global__ void __launch_bounds__(256) attn_bwd_dq_fixed_kernel(const float* __restrict__ q, const float* __restrict__ kh,
                                                                const float* __restrict__ dS,
                                                                const float* __restrict__ q_scale, float* __restrict__ dq,
                                                                const float* __restrict__ pre,
                                                                float* __restrict__ scale_part, AttnBwdGeom g) {
  attn_bwd_dq_body(q, kh, dS, q_scale, dq, nullptr, pre, scale_part, g);
}

// one warp per (sequence, head, key j in [0, nkt)): dkh = 8 * sum_i dS[i,j] qh[i,:], dvv = sum_i P[i,j] dO[i,:]
// scale_part / null_part (deterministic mode, else NULL): the CTA's k_scale sum goes to its slot blockIdx.x, and the
// null keys / values of sequence bi to slot bi, instead of dk_scale / dnull_kv
__device__ __forceinline__ void attn_bwd_dkv_body(const float* __restrict__ kv, const float* __restrict__ null_kv,
                                                  const float* __restrict__ qh, const float* __restrict__ dO,
                                                  const float* __restrict__ P, const float* __restrict__ dS,
                                                  const float* __restrict__ k_scale, float* __restrict__ dkv,
                                                  float* __restrict__ dnull_kv, float* __restrict__ dk_scale,
                                                  const float* __restrict__ preK, const float* __restrict__ preV,
                                                  const AttnBwdGeom& g, float* __restrict__ scale_part,
                                                  float* __restrict__ null_part) {
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
      const int64_t nidx = ((int64_t)h * 2 * g.nnull + 2 * j) * g.dh;
      if (null_part) {  // deterministic mode: sequence bi's terms to slot bi
        float* nk = null_part + (int64_t)bi * g.H * 2 * g.nnull * g.dh + nidx;
#pragma unroll
        for (int c = 0; c < kDPL; ++c) { const int d = lane + 32 * c; if (d < g.dh) { nk[d] = draw[c]; nk[g.dh + d] = av[c]; } }
      } else {
        float* nk = dnull_kv + nidx;
#pragma unroll
        for (int c = 0; c < kDPL; ++c) {
          const int d = lane + 32 * c;
          if (d < g.dh) { atomicAdd(nk + d, draw[c]); atomicAdd(nk + g.dh + d, av[c]); }
        }
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
    if (scale_part) scale_part[(int64_t)blockIdx.x * g.dh + threadIdx.x] = a;
    else atomicAdd(dk_scale + threadIdx.x, a);
  }
}
__global__ void __launch_bounds__(256) attn_bwd_dkv_kernel(const float* __restrict__ kv, const float* __restrict__ null_kv,
                                                           const float* __restrict__ qh, const float* __restrict__ dO,
                                                           const float* __restrict__ P, const float* __restrict__ dS,
                                                           const float* __restrict__ k_scale, float* __restrict__ dkv,
                                                           float* __restrict__ dnull_kv, float* __restrict__ dk_scale,
                                                           const float* __restrict__ preK, const float* __restrict__ preV,
                                                           AttnBwdGeom g) {
  attn_bwd_dkv_body(kv, null_kv, qh, dO, P, dS, k_scale, dkv, dnull_kv, dk_scale, preK, preV, g, nullptr, nullptr);
}
__global__ void __launch_bounds__(256) attn_bwd_dkv_fixed_kernel(const float* __restrict__ kv,
                                                                 const float* __restrict__ null_kv,
                                                                 const float* __restrict__ qh, const float* __restrict__ dO,
                                                                 const float* __restrict__ P, const float* __restrict__ dS,
                                                                 const float* __restrict__ k_scale, float* __restrict__ dkv,
                                                                 const float* __restrict__ preK,
                                                                 const float* __restrict__ preV, AttnBwdGeom g,
                                                                 float* __restrict__ scale_part,
                                                                 float* __restrict__ null_part) {
  attn_bwd_dkv_body(kv, null_kv, qh, dO, P, dS, k_scale, dkv, nullptr, nullptr, preK, preV, g, scale_part, null_part);
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

// The attention backward's scratch, per (sequence, head): qh [n, dh], kh and vv [nkt, dh], P and dS [n, nkt], then the
// batched-product outputs preQ = dS.kh [n, dh], preK = dS^T.qh and preV = P^T.dO [nkt, dh].  attention_forward_dropout
// uses the first four.
struct AttnBwdBufs { float *qh, *kh, *vv, *P, *dS, *preQ, *preK, *preV; };

AttnBwdBufs attn_bwd_bufs(float* scratch, const AttnBwdGeom& g) {
  const int64_t bh = (int64_t)g.b * g.H, nkt = g.nnull + g.m;
  AttnBwdBufs B;
  B.qh = scratch;
  B.kh = B.qh + bh * g.n * g.dh;
  B.vv = B.kh + bh * nkt * g.dh;
  B.P = B.vv + bh * nkt * g.dh;
  B.dS = B.P + bh * g.n * nkt;
  B.preQ = B.dS + bh * g.n * nkt;
  B.preK = B.preQ + bh * g.n * g.dh;
  B.preV = B.preK + bh * nkt * g.dh;
  return B;
}

// Deterministic-mode scratch of attention_backward: the larger of the dq kernel's slots and the dkv kernel's (k_scale and
// null_kv), each followed by colsum_fixed's partials over its CTA slots
int64_t attn_bwd_det_floats(const AttnBwdGeom& g) {
  const int64_t bh = (int64_t)g.b * g.H, nq = (bh * g.n + 7) / 8, nk = (bh * (g.nnull + g.m) + 7) / 8;
  const int64_t fq = nq * g.dh + colsum_fixed_floats(nq, g.dh);
  const int64_t fk = nk * g.dh + (int64_t)g.b * g.H * 2 * g.nnull * g.dh + colsum_fixed_floats(nk, g.dh);
  return fq > fk ? fq : fk;
}

int64_t attn_bwd_scratch_floats(int b, int H, int n, int nkt, int dh) {
  // everything attn_bwd_bufs carves: 2 [n, dh] + 4 [nkt, dh] + 2 [n, nkt] per (sequence, head)
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
  const AttnBwdBufs B = attn_bwd_bufs(scratch, g);
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
    preQ = B.preQ;
    preK = B.preK;
    preV = B.preV;
    const GemmBatch bq{(int)bh, 1, (int64_t)g.n * nkt, 0, (int64_t)nkt * g.dh, 0, (int64_t)g.n * g.dh, 0};
    PHK_TRY(sgemm_batched(B.dS, nkt, 1, B.kh, g.dh, 1, preQ, g.dh, g.n, g.dh, nkt, 0, bq, st, bf16_products));  // dS . kh
    const GemmBatch bk{(int)bh, 1, (int64_t)g.n * nkt, 0, (int64_t)g.n * g.dh, 0, (int64_t)nkt * g.dh, 0};
    PHK_TRY(sgemm_batched(B.dS, 1, nkt, B.qh, g.dh, 1, preK, g.dh, nkt, g.dh, g.n, 0, bk, st, bf16_products));  // dS^T . qh
    const GemmBatch bv{(int)bh, g.H, (int64_t)g.H * g.n * nkt, (int64_t)g.n * nkt, (int64_t)g.n * I, (int64_t)g.dh,
                       (int64_t)g.H * nkt * g.dh, (int64_t)nkt * g.dh};
    PHK_TRY(sgemm_batched(B.P, 1, nkt, dO, I, 1, preV, g.dh, nkt, g.dh, g.n, 0, bv, st, bf16_products));     // P^T . dO
  }
  const int64_t nq = (bh * g.n + 7) / 8, nk = (bh * nkt + 7) / 8;  // CTAs of the dq and dkv kernels
  if (t_det.p) {
    // deterministic mode: each CTA's q_scale / k_scale sum and each sequence's null_kv terms go to their own slots, which
    // are then added in order (the dq slots are dead before the dkv kernel reuses the region)
    PHK_REQUIRE(attn_bwd_det_floats(g) <= t_det.floats, PHK_E_WORKSPACE, "train: deterministic reduction scratch too small");
    float* qs = t_det.p;
    PHK_KERNEL_LAUNCH(attn_bwd_dq_fixed_kernel, dim3((unsigned)nq), dim3(256), (size_t)(0), st, q, B.kh, B.dS, A.q_scale, dq, (const float*)preQ, qs, g);
    PHK_LAUNCH_CHECK();
    PHK_TRY(colsum_fixed(qs, nq, g.dh, g.dh, (float*)G.q_scale, qs + nq * g.dh, t_det.floats - nq * g.dh, st));
    float* ks = t_det.p;
    float* ns = g.nnull ? ks + nk * g.dh : nullptr;
    const int64_t nnf = (int64_t)g.H * 2 * g.nnull * g.dh;  // null_kv floats
    PHK_KERNEL_LAUNCH(attn_bwd_dkv_fixed_kernel, dim3((unsigned)nk), dim3(256), (size_t)(0), st, kv, A.null_kv, B.qh, dO, B.P, B.dS, A.k_scale, dkv,
                      (const float*)preK, (const float*)preV, g, ks, ns);
    PHK_LAUNCH_CHECK();
    if (ns) PHK_TRY(add_slots(ns, g.b, nnf, (float*)G.null_kv, st));
    const int64_t used = nk * g.dh + (ns ? g.b * nnf : 0);
    PHK_TRY(colsum_fixed(ks, nk, g.dh, g.dh, (float*)G.k_scale, t_det.p + used, t_det.floats - used, st));
  } else {
    PHK_KERNEL_LAUNCH(attn_bwd_dq_kernel, dim3((unsigned)nq), dim3(256), (size_t)(0), st, q, B.kh, B.dS, A.q_scale, dq, (float*)G.q_scale, (const float*)preQ, g);
    PHK_LAUNCH_CHECK();
    PHK_KERNEL_LAUNCH(attn_bwd_dkv_kernel, dim3((unsigned)nk), dim3(256), (size_t)(0), st, kv, A.null_kv, B.qh, dO, B.P, B.dS, A.k_scale, dkv,
                      (float*)G.null_kv, (float*)G.k_scale, (const float*)preK, (const float*)preV, g);
    PHK_LAUNCH_CHECK();
  }
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
  const AttnBwdBufs B = attn_bwd_bufs(scratch, g);
  float *qh = B.qh, *kh = B.kh, *vv = B.vv, *P = B.P;
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
// part (deterministic mode, else NULL): the chunk's sums go to its slot [blockIdx.y][D][27] instead of dw
__device__ __forceinline__ void peg_bwd_dw_body(const float* __restrict__ x, const float* __restrict__ dy,
                                                float* __restrict__ dw, int64_t P, int T, int H, int W, int D, int pad_t0,
                                                float* __restrict__ part) {
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
    if (d >= D) continue;
    if (part) part[(int64_t)blockIdx.y * 27 * D + (int64_t)d * 27 + tap] = p1 > p0 ? acc[j] : 0.f;
    else if (p1 > p0) atomicAdd(dw + (int64_t)d * 27 + tap, acc[j]);  // dsconv.weight[d, 0, kt, kh, kw]
  }
}
__global__ void __launch_bounds__(128) peg_bwd_dw_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                         float* __restrict__ dw, int64_t P, int T, int H, int W, int D,
                                                         int pad_t0) {
  peg_bwd_dw_body(x, dy, dw, P, T, H, W, D, pad_t0, nullptr);
}
__global__ void __launch_bounds__(128) peg_bwd_dw_fixed_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                               int64_t P, int T, int H, int W, int D, int pad_t0,
                                                               float* __restrict__ part) {
  peg_bwd_dw_body(x, dy, nullptr, P, T, H, W, D, pad_t0, part);
}

inline int64_t peg_det_floats(int64_t D) { return PEG_DW_CHUNKS * 27 * D; }

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

// Deterministic mode, token embedding: the rows of one id are summed in row order by one CTA, the one of the id's first
// row (the leader).  CTA r first looks for an earlier row with its id and leaves if there is one; the leader then walks
// the rows after it in tiles of blockDim.x, lists the tile's matching rows in order (a prefix sum over the tile) and adds
// their dx rows, columns over threads, into four accumulators taken in turn (a0 gets the entry, then the four rotate).
__device__ __forceinline__ int64_t embed_row_id(const int64_t* ids, int64_t r, int vocab_rows) {
  const int64_t id = ids[r];
  return id < 0 ? 0 : (id >= vocab_rows ? vocab_rows - 1 : id);
}
__global__ void __launch_bounds__(128) embed_tok_fixed_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dx,
                                                              float* __restrict__ dtok, int64_t rows, int dim, float alpha,
                                                              int vocab_rows) {
  __shared__ int found;
  __shared__ int scan[128];
  __shared__ int64_t list[128];
  const int t = threadIdx.x;
  const int64_t r = blockIdx.x;
  const int64_t id = embed_row_id(ids, r, vocab_rows);
  if (t == 0) found = 0;
  __syncthreads();
  for (int64_t q = t; q < r; q += blockDim.x)
    if (embed_row_id(ids, q, vocab_rows) == id) { found = 1; break; }
  __syncthreads();
  if (found) return;  // uniform over the CTA
  for (int c0 = 0; c0 < dim; c0 += 128 * 4) {
    float a0[4], a1[4], a2[4], a3[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) a0[j] = a1[j] = a2[j] = a3[j] = 0.f;
    for (int64_t base = r; base < rows; base += blockDim.x) {
      const int64_t q = base + t;
      const int hit = q < rows && embed_row_id(ids, q, vocab_rows) == id;
      scan[t] = hit;
      __syncthreads();
      for (int off = 1; off < 128; off <<= 1) {  // inclusive prefix sum over the tile
        const int v = t >= off ? scan[t - off] : 0;
        __syncthreads();
        scan[t] += v;
        __syncthreads();
      }
      if (hit) list[scan[t] - 1] = q;
      const int cnt = scan[127];
      __syncthreads();
      for (int e = 0; e < cnt; ++e) {
        const float* xr = dx + list[e] * dim;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = c0 + t + 128 * j;
          const float v = a0[j] + (c < dim ? alpha * xr[c] : 0.f);
          a0[j] = a1[j]; a1[j] = a2[j]; a2[j] = a3[j]; a3[j] = v;
        }
      }
      __syncthreads();  // list and scan are rewritten by the next tile
    }
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + t + 128 * j;
      if (c < dim) dtok[id * dim + c] += (a0[j] + a1[j]) + (a2[j] + a3[j]);
    }
  }
}
// Deterministic mode, position embedding: dpos[p, c] += sum over the sequences b, in order, of alpha dx[b n + p, c]
__global__ void embed_pos_fixed_kernel(const float* __restrict__ dx, float* __restrict__ dpos, int64_t rows, int n, int dim,
                                       float alpha) {
  const int64_t total = (int64_t)n * dim, nb = rows / n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float a = 0.f;
    for (int64_t b = 0; b < nb; ++b) a += alpha * dx[b * total + i];
    dpos[i] += a;
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

// Deterministic mode: dtable[u, h] = sum of dbias[h, i, j] over the (i, j) pairs with delta u, in increasing i (a gather:
// the pairs of u are i = j + delta with both inside the grid)
__global__ void cpb_dtable_fixed_kernel(const float* __restrict__ dbias, float* __restrict__ dtable, int heads, int d0,
                                        int d1, int d2) {
  const int n = d0 * d1 * d2;
  const int64_t total = (int64_t)n * n;
  const int s1 = 2 * d1 - 1, s2 = 2 * d2 - 1;
  const int64_t U = (int64_t)(2 * d0 - 1) * s1 * s2;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < U * heads; idx += (int64_t)gridDim.x * blockDim.x) {
    const int h = (int)(idx % heads);
    const int u = (int)(idx / heads);
    const int e0 = u / (s1 * s2) - (d0 - 1), e1 = (u / s2) % s1 - (d1 - 1), e2 = u % s2 - (d2 - 1);  // i - j per axis
    float a = 0.f;
    for (int i0 = e0 > 0 ? e0 : 0; i0 < d0 && i0 - e0 < d0; ++i0)
      for (int i1 = e1 > 0 ? e1 : 0; i1 < d1 && i1 - e1 < d1; ++i1)
        for (int i2 = e2 > 0 ? e2 : 0; i2 < d2 && i2 - e2 < d2; ++i2) {
          const int64_t i = ((int64_t)i0 * d1 + i1) * d2 + i2, j = ((int64_t)(i0 - e0) * d1 + (i1 - e1)) * d2 + (i2 - e2);
          a += dbias[(int64_t)h * total + i * n + j];
        }
    dtable[idx] = a;
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
  if (t_det.p) {
    PHK_KERNEL_LAUNCH(cpb_dtable_fixed_kernel, dim3(ew_grid(U * H)), dim3(256), (size_t)(0), st, dbias, dtable, H, d0, d1, d2);
    PHK_LAUNCH_CHECK();
  } else {
    PHK_CUDA(cudaMemsetAsync(dtable, 0, U * H * sizeof(float), st));
    const int64_t nn = (int64_t)d0 * d1 * d2 * d0 * d1 * d2;
    PHK_KERNEL_LAUNCH(cpb_dtable_kernel, dim3(ew_grid(nn)), dim3(256), (size_t)(0), st, dbias, dtable, H, d0, d1, d2);
    PHK_LAUNCH_CHECK();
  }
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

// Data-parallel overlap (SURVEY 8e): the caller may hand in CUDA events that the NEXT phk_maskgit_train_step or
// phk_cvivit_backward call of this thread records on its stream as groups of gradients become final -- for the MaskGit
// step events[0]: the head + norm_out, events[1 + k]: transformer layer depth-1-k (backward order), events[depth + 1]:
// embeddings + position-bias MLP = everything; for C-ViViT see phk_cvivit_backward_progress_groups.  A side stream can
// then all-reduce each finished slice of the flat gradient bucket while the layers below still run.
static thread_local void** g_progress_events = nullptr;
static thread_local int g_progress_count = 0;
extern "C" int phk_train_set_progress_events(void** events, int32_t count) {
  g_progress_events = events;
  g_progress_count = events ? count : 0;
  return 0;
}
// See include/phk.h: the deterministic mode of this thread's next backward calls and workspace queries
extern "C" int32_t phk_train_set_deterministic(int32_t on) {
  const int32_t prev = t_det_mode;
  t_det_mode = on ? 1 : 0;
  return prev;
}
static inline int progress_mark(void** ev, int n, int idx, cudaStream_t st) {
  if (ev && idx < n && ev[idx]) PHK_CUDA(cudaEventRecord(reinterpret_cast<cudaEvent_t>(ev[idx]), st));
  return 0;
}

// The progress events of one C-ViViT backward, recorded in order: each progress_next closes the next group.  A NULL
// Progress (the entry points that take no events) records nothing.
struct Progress {
  void** ev = nullptr;
  int n = 0, next = 0;
};
static inline int progress_next(Progress* p, cudaStream_t st) {
  return p ? progress_mark(p->ev, p->n, p->next++, st) : 0;
}

// ------------------------------------------------------------------------------------------------------------------
// The three stages of one differentiation of the MaskGit / TokenCritic body, shared by phk_maskgit_train_step (a loss
// head) and phk_maskgit_backward (a gradient the caller supplies):
//   1. step_forward   embed -> [PEG, self-attn, cross-attn, FF] x depth -> norm_out, keeping every layer's activations;
//                     S.emb = the final embeddings [R, D]
//   2. the head       (in each entry point) accumulates the head's parameter gradients and writes d/d(emb) to S.dtmp
//   3. step_backward  norm_out, transformer, embedding and position-bias backward from S.dtmp
// ------------------------------------------------------------------------------------------------------------------
namespace phk {
namespace {

struct Step {
  const phk_maskgit_t* m = nullptr;
  const phk_maskgit_t* grads = nullptr;
  const phk_transformer_t* T = nullptr;
  const phk_transformer_t* GT = nullptr;
  const int64_t* ids = nullptr;
  int b = 0, n = 0, pt = 0, ph = 0, pw = 0, L = 0;
  const float* context = nullptr;
  const uint8_t* text_mask = nullptr;
  const uint8_t* video_mask = nullptr;
  int prec = PHK_PREC_F32;
  phk_stream_t s = nullptr;
  cudaStream_t st = nullptr;
  const phk_dropout_t* dropout = nullptr;
  bool drop_on = false;
  float attn_p = 0.f, ff_p = 0.f;
  int D = 0, H = 0, DH = 0, I = 0;
  int64_t R = 0, CR = 0;
  Arena ar{nullptr, 0, 0};
  TcScratch tc{nullptr, nullptr, 0};
  float* emb = nullptr;
  float* bias = nullptr;
  float* dbias = nullptr;
  float* asc = nullptr;
  const float* xf = nullptr;
  float* dxa = nullptr;
  float* dxb = nullptr;
  float* dtmp = nullptr;
  float2* stats = nullptr;
  LayerSave* sv = nullptr;
  uint64_t (*bases)[3] = nullptr;
  ~Step() { delete[] sv; delete[] bases; }

  // dropout: site k of layer l (0 self-attention, 1 cross-attention, 2 FF) draws from counters offset + bases[l][k];
  // p == 0: the site is off
  DropSite site(float p, int l, int k) const {
    DropSite d{0.f, 0.f, 0u, 0u, 0u};
    if (drop_on && p > 0.f) {
      d.p = p; d.scale = 1.0f / (1.0f - p);
      d.k0 = (uint32_t)dropout->seed; d.k1 = (uint32_t)(dropout->seed >> 32);
      d.base = dropout->offset + bases[l][k];
    }
    return d;
  }
};

// Fills the derived members of S from its inputs (m, grads, b, n, L, context, prec, s, dropout, workspace arena).
void step_init(Step& S) {
  S.T = &S.m->transformer;
  S.GT = &S.grads->transformer;
  S.st = to_stream(S.s);
  S.drop_on = S.dropout && (S.dropout->attn_p > 0.f || S.dropout->ff_p > 0.f);
  S.attn_p = S.dropout ? S.dropout->attn_p : 0.f;
  S.ff_p = S.dropout ? S.dropout->ff_p : 0.f;
  S.D = S.m->dim; S.H = S.T->heads; S.DH = S.T->dim_head; S.I = S.H * S.DH;
  S.R = (int64_t)S.b * S.n; S.CR = (int64_t)S.b * S.L;
}

// ------------------------------------------------------------------------------------------------------------------
// One transformer layer (attention.py:311-330): forward keeping its activations, and backward.  Shared by every stack
// whose sequences are runs of n contiguous rows: MaskGit / TokenCritic (b videos of n tokens, PEG over (pt, ph, pw),
// cross-attention to the text) and the stacks of the C-ViViT encoder and decoder (phk_cvivit_backward,
// phk_cvivit_decode_backward).
// ------------------------------------------------------------------------------------------------------------------
struct LayerCall {
  const phk_transformer_t* T = nullptr;    // weights
  const phk_transformer_t* GT = nullptr;   // gradient table of the same layout
  int b = 0, n = 0;                        // b sequences of n contiguous rows
  int pegB = 0, pegT = 0, pegH = 0, pegW = 0;  // video shape the layers' PEG runs over (layout 0 on the rows)
  const float* bias = nullptr;             // self-attention additive bias [H, n, n], or NULL
  float* dbias = nullptr;                  // its gradient, accumulated (NULL: the bias is a constant)
  const uint8_t* key_mask = nullptr;       // self-attention key mask [b, n], or NULL
  const float* context = nullptr;          // cross-attention context [b, L, dim_context], or NULL
  int L = 0;
  const uint8_t* text_mask = nullptr;      // [b, L]
  int prec = PHK_PREC_F32;
  phk_stream_t s = nullptr;
  cudaStream_t st = nullptr;
  TcScratch tc{nullptr, nullptr, 0};
  float* asc = nullptr;                    // attention scratch: attn_bwd_scratch_floats of the larger attention
};

// Gradient scratch of layer_backward: dtmp [R, D], dq [R, I], dkv [R, 2I], dob [R, I], dh [R, 2 inner], dg [R, inner],
// dckv [CR, 2I] / dctxn [CR, dim_context] (cross-attention only), LayerNorm statistics [max(R, CR)]
struct LayerGrads { float *dtmp, *dq, *dkv, *dob, *dh, *dg, *dckv, *dctxn; float2* stats; };

// Layer l of c.T on x0 [R, D]: every activation the backward reads is kept in Sv, the output lands in *xout (fresh).
int layer_forward(const LayerCall& c, int l, const float* x0, LayerSave& Sv, float** xout, Arena& ar,
                  const DropSite& d_self, const DropSite& d_cross, const DropSite& d_ff) {
  const phk_transformer_t* T = c.T;
  const phk_layer_t& Ly = T->layers[l];
  const int b = c.b, n = c.n, L = c.L;
  const int D = T->dim, H = T->heads, DH = T->dim_head, I = H * DH;
  const int64_t R = (int64_t)b * n, CR = (int64_t)b * L;
  const int prec = c.prec;
  const phk_stream_t s = c.s;
  const cudaStream_t st = c.st;
  const TcScratch& tc = c.tc;
  std::memset(&Sv, 0, sizeof(Sv));
  const int inner = Ly.ff.inner;
  Sv.x0 = const_cast<float*>(x0);
  Sv.x1 = Ly.has_peg ? ar.f(R * D) : Sv.x0;  // without PEG the self-attention reads x0
  Sv.xn1 = ar.f(R * D); Sv.q1 = ar.f(R * I); Sv.kv1 = ar.f(R * 2 * I); Sv.o1 = ar.f(R * I);
  Sv.x2 = ar.f(R * D); Sv.x3 = ar.f(R * D); Sv.xn3 = ar.f(R * D); Sv.h = ar.f(R * 2 * (int64_t)inner); Sv.g = ar.f(R * (int64_t)inner);
  *xout = ar.f(R * D);
  PHK_REQUIRE(Sv.x1 && Sv.xn1 && Sv.q1 && Sv.kv1 && Sv.o1 && Sv.x2 && Sv.x3 && Sv.xn3 && Sv.h && Sv.g && *xout, PHK_E_WORKSPACE,
              "train: workspace too small (activations)");
  // x1 = peg(x0) + x0
  if (Ly.has_peg) {
    PHK_REQUIRE((int64_t)c.pegB * c.pegT * c.pegH * c.pegW == R, PHK_E_SHAPE, "train: PEG shape does not cover the rows");
    PHK_TRY(phk_peg3d(Sv.x0, Ly.peg.w, Ly.peg.b, Sv.x1, c.pegB, c.pegT, c.pegH, c.pegW, D, Ly.peg.causal, 0, s));
  }
  // self attention: q from LN(x1), k/v from RAW x1 (attention.py:140-144)
  const phk_attn_t& A = Ly.self_attn;
  phk_attn_geom_t ag;
  PHK_TRY(phk_layernorm(Sv.x1, A.norm_g, A.norm_b, Sv.xn1, nullptr, R, D, 0, 0, 0, 0, s));
  PHK_TRY(linear_fwd(prec, tc, Sv.xn1, A.wq, Sv.q1, R, I, D, nullptr, nullptr, s));
  PHK_TRY(linear_fwd(prec, tc, Sv.x1, A.wkv, Sv.kv1, R, 2 * I, D, nullptr, nullptr, s));
  std::memset(&ag, 0, sizeof(ag));
  ag.n_outer = b; ag.n_inner = 1; ag.n_q = n; ag.n_k = n; ag.heads = H; ag.dim_head = DH; ag.num_null_kv = A.num_null_kv;
  ag.q_outer = (int64_t)n * I; ag.q_tok = I; ag.k_outer = (int64_t)n * 2 * I; ag.k_tok = 2 * I;
  ag.o_outer = ag.q_outer; ag.o_tok = I; ag.mask_off_from = -1; ag.scale = 8.f;
  PHK_REQUIRE(A.num_null_kv == 0, PHK_E_UNSUPPORTED, "train: self-attention null-kv is not supported");
  if (d_self.p > 0.f) {
    const AttnBwdGeom g1{b, H, n, n, 0, DH};
    PHK_TRY(attention_forward_dropout(Sv.q1, Sv.kv1, A, c.bias, c.key_mask, Sv.o1, g1, c.asc, st, d_self));
  } else {
    PHK_TRY(phk_attention(Sv.q1, Sv.kv1, A.null_kv, A.q_scale, A.k_scale, c.bias, c.key_mask, nullptr, Sv.o1, &ag, s));
  }
  PHK_TRY(linear_fwd(prec, tc, Sv.o1, A.wo, Sv.x2, R, D, I, nullptr, Sv.x1, s));  // x2 = x1 + o Wo^T
  if (Ly.has_cross && c.context) {
    const phk_attn_t& Cx = Ly.cross_attn;
    const int dc = Cx.dim_context;
    Sv.ctxn = ar.f(CR * dc); Sv.ckv = ar.f(CR * 2 * I); Sv.xn2 = ar.f(R * D); Sv.q2 = ar.f(R * I); Sv.o2 = ar.f(R * I);
    PHK_REQUIRE(Sv.ctxn && Sv.ckv && Sv.xn2 && Sv.q2 && Sv.o2, PHK_E_WORKSPACE, "train: workspace too small (cross)");
    PHK_TRY(phk_layernorm(c.context, Cx.ctx_g, Cx.ctx_b, Sv.ctxn, nullptr, CR, dc, 0, 0, 0, 0, s));
    PHK_TRY(linear_fwd(prec, tc, Sv.ctxn, Cx.wkv, Sv.ckv, CR, 2 * I, dc, nullptr, nullptr, s));
    PHK_TRY(phk_layernorm(Sv.x2, Cx.norm_g, Cx.norm_b, Sv.xn2, nullptr, R, D, 0, 0, 0, 0, s));
    PHK_TRY(linear_fwd(prec, tc, Sv.xn2, Cx.wq, Sv.q2, R, I, D, nullptr, nullptr, s));
    std::memset(&ag, 0, sizeof(ag));
    ag.n_outer = b; ag.n_inner = 1; ag.n_q = n; ag.n_k = L; ag.heads = H; ag.dim_head = DH; ag.num_null_kv = Cx.num_null_kv;
    ag.q_outer = (int64_t)n * I; ag.q_tok = I; ag.k_outer = (int64_t)L * 2 * I; ag.k_tok = 2 * I;
    ag.o_outer = ag.q_outer; ag.o_tok = I; ag.kv_outer_mod = b; ag.mask_outer_mod = b; ag.mask_off_from = -1; ag.scale = 8.f;
    if (d_cross.p > 0.f) {
      PHK_REQUIRE(Cx.num_null_kv <= 8, PHK_E_UNSUPPORTED, "train: more than 8 null key/values");
      const AttnBwdGeom g2{b, H, n, L, Cx.num_null_kv, DH};
      PHK_TRY(attention_forward_dropout(Sv.q2, Sv.ckv, Cx, nullptr, c.text_mask, Sv.o2, g2, c.asc, st, d_cross));
    } else {
      PHK_TRY(phk_attention(Sv.q2, Sv.ckv, Cx.null_kv, Cx.q_scale, Cx.k_scale, nullptr, c.text_mask, nullptr, Sv.o2, &ag, s));
    }
    PHK_TRY(linear_fwd(prec, tc, Sv.o2, Cx.wo, Sv.x3, R, D, I, nullptr, Sv.x2, s));  // x3 = x2 + o2 Wo^T
  } else {
    PHK_CUDA(cudaMemcpyAsync(Sv.x3, Sv.x2, R * D * 4, cudaMemcpyDeviceToDevice, st));
  }
  // feed forward (attention.py:45-53)
  PHK_TRY(phk_layernorm(Sv.x3, Ly.ff.ln_g, Ly.ff.ln_b, Sv.xn3, nullptr, R, D, 0, 0, 0, 0, s));
  PHK_TRY(linear_fwd(prec, tc, Sv.xn3, Ly.ff.w1, Sv.h, R, 2 * inner, D, nullptr, nullptr, s));
  if (d_ff.p > 0.f) {
    PHK_KERNEL_LAUNCH(geglu_dropout_kernel, dim3(ew_grid_fwd(R * inner)), dim3(256), (size_t)(0), st, Sv.h, Sv.g, R, inner, d_ff);
    PHK_LAUNCH_CHECK();
  } else {
    PHK_TRY(phk_geglu(Sv.h, Sv.g, R, inner, s));
  }
  return linear_fwd(prec, tc, Sv.g, Ly.ff.w2, *xout, R, D, inner, nullptr, Sv.x3, s);  // x4 = x3 + g W2^T
}

// Backward of layer l: on entry *dx holds d/d(layer output), on return d/d(x0) (*dx and *dx_alt may swap).  Parameter
// gradients accumulate into c.GT, the bias gradient into c.dbias; d_context (optional) accumulates d/d(context).
int layer_backward(const LayerCall& c, int l, const LayerSave& Sv, float** dx, float** dx_alt, const LayerGrads& G,
                   float* d_context, const DropSite& d_self, const DropSite& d_cross, const DropSite& d_ff) {
  const phk_transformer_t* T = c.T;
  const phk_layer_t& Ly = T->layers[l];
  const phk_layer_t& Gy = c.GT->layers[l];
  const int b = c.b, n = c.n, L = c.L;
  const int D = T->dim, H = T->heads, DH = T->dim_head, I = H * DH;
  const int64_t R = (int64_t)b * n, CR = (int64_t)b * L;
  const int prec = c.prec;
  const phk_stream_t s = c.s;
  const cudaStream_t st = c.st;
  const TcScratch& tc = c.tc;
  const int inner = Ly.ff.inner;
  float* d = *dx;
  // feed forward: x4 = x3 + geglu(LN(x3) W1^T) W2^T
  PHK_TRY(dgrad_p(prec, tc, d, Ly.ff.w2, G.dg, R, D, inner, 0, s));
  PHK_TRY(wgrad_p(prec, tc, d, Sv.g, (float*)Gy.ff.w2, R, D, inner, s));
  PHK_KERNEL_LAUNCH(geglu_bwd_kernel, dim3(ew_grid(R * inner)), dim3(256), (size_t)(0), st, Sv.h, G.dg, G.dh, R, inner, d_ff);
  PHK_LAUNCH_CHECK();
  PHK_TRY(wgrad_p(prec, tc, G.dh, Sv.xn3, (float*)Gy.ff.w1, R, 2 * inner, D, s));
  PHK_TRY(dgrad_p(prec, tc, G.dh, Ly.ff.w1, G.dtmp, R, 2 * inner, D, 0, s));
  PHK_TRY(ln_backward(Sv.x3, Ly.ff.ln_g, G.dtmp, d, 1, (float*)Gy.ff.ln_g, (float*)Gy.ff.ln_b, G.stats, R, D, st));
  // cross attention: x3 = x2 + attn(LN(x2) Wq^T, LN_ctx(context) Wkv^T) Wo^T
  if (Sv.o2) {
    const phk_attn_t& Cx = Ly.cross_attn;
    const phk_attn_t& Gx = Gy.cross_attn;
    const int dc = Cx.dim_context;
    PHK_REQUIRE(Cx.num_null_kv <= 8, PHK_E_UNSUPPORTED, "train: more than 8 null key/values");
    PHK_TRY(dgrad_p(prec, tc, d, Cx.wo, G.dob, R, D, I, 0, s));
    PHK_TRY(wgrad_p(prec, tc, d, Sv.o2, (float*)Gx.wo, R, D, I, s));
    const AttnBwdGeom g2{b, H, n, L, Cx.num_null_kv, DH};
    PHK_TRY(attention_backward(Sv.q2, Sv.ckv, Cx, Gx, nullptr, c.text_mask, G.dob, G.dq, G.dckv, nullptr, g2, c.asc, st,
                               prec == PHK_PREC_BF16, d_cross));
    PHK_TRY(wgrad_p(prec, tc, G.dq, Sv.xn2, (float*)Gx.wq, R, I, D, s));
    PHK_TRY(dgrad_p(prec, tc, G.dq, Cx.wq, G.dtmp, R, I, D, 0, s));
    PHK_TRY(ln_backward(Sv.x2, Cx.norm_g, G.dtmp, d, 1, (float*)Gx.norm_g, nullptr, G.stats, R, D, st));
    PHK_TRY(wgrad_p(prec, tc, G.dckv, Sv.ctxn, (float*)Gx.wkv, CR, 2 * I, dc, s));
    PHK_TRY(dgrad_p(prec, tc, G.dckv, Cx.wkv, G.dctxn, CR, 2 * I, dc, 0, s));
    // context_norm backward: d/d(context) accumulates over the layers when the caller asks for it
    PHK_TRY(ln_backward(c.context, Cx.ctx_g, G.dctxn, d_context, d_context ? 1 : 0, (float*)Gx.ctx_g, nullptr, G.stats, CR, dc, st));
  }
  // self attention: x2 = x1 + attn(LN(x1) Wq^T, x1 Wkv^T) Wo^T
  {
    const phk_attn_t& A = Ly.self_attn;
    const phk_attn_t& GA = Gy.self_attn;
    PHK_TRY(dgrad_p(prec, tc, d, A.wo, G.dob, R, D, I, 0, s));
    PHK_TRY(wgrad_p(prec, tc, d, Sv.o1, (float*)GA.wo, R, D, I, s));
    const AttnBwdGeom g1{b, H, n, n, 0, DH};
    PHK_TRY(attention_backward(Sv.q1, Sv.kv1, A, GA, c.bias, c.key_mask, G.dob, G.dq, G.dkv, c.dbias, g1, c.asc, st,
                               prec == PHK_PREC_BF16, d_self));
    PHK_TRY(wgrad_p(prec, tc, G.dq, Sv.xn1, (float*)GA.wq, R, I, D, s));
    PHK_TRY(wgrad_p(prec, tc, G.dkv, Sv.x1, (float*)GA.wkv, R, 2 * I, D, s));
    PHK_TRY(dgrad_p(prec, tc, G.dq, A.wq, G.dtmp, R, I, D, 0, s));
    PHK_TRY(ln_backward(Sv.x1, A.norm_g, G.dtmp, d, 1, (float*)GA.norm_g, nullptr, G.stats, R, D, st));
    PHK_TRY(dgrad_p(prec, tc, G.dkv, A.wkv, d, R, 2 * I, D, 1, s));  // the raw-x path of k, v
  }
  if (!Ly.has_peg) return 0;  // x1 = x0
  // PEG: x1 = x0 + conv(x0) + b
  PHK_TRY(colsum(d, R, D, D, (float*)Gy.peg.b, st));
  PHK_REQUIRE(D <= 128 * PEG_DW_MAXJ, PHK_E_UNSUPPORTED, "train: PEG backward needs dim <= 1024");
  if (t_det.p) {  // deterministic mode: one [D, 27] slot per chunk of positions, added in order
    PHK_REQUIRE(peg_det_floats(D) <= t_det.floats, PHK_E_WORKSPACE, "train: deterministic reduction scratch too small");
    PHK_KERNEL_LAUNCH(peg_bwd_dw_fixed_kernel, dim3(27, PEG_DW_CHUNKS), dim3(128), (size_t)(0), st, Sv.x0, (const float*)d, R, c.pegT, c.pegH, c.pegW, D, Ly.peg.causal ? 2 : 1, t_det.p);
    PHK_LAUNCH_CHECK();
    PHK_TRY(add_slots(t_det.p, PEG_DW_CHUNKS, 27 * (int64_t)D, (float*)Gy.peg.w, st));
  } else {
    PHK_KERNEL_LAUNCH(peg_bwd_dw_kernel, dim3(27, PEG_DW_CHUNKS), dim3(128), (size_t)(0), st, Sv.x0, d, (float*)Gy.peg.w, R, c.pegT, c.pegH, c.pegW, D, Ly.peg.causal ? 2 : 1);
    PHK_LAUNCH_CHECK();
  }
  PHK_KERNEL_LAUNCH(peg_bwd_kernel, dim3((unsigned)R), dim3(128), (size_t)(0), st, Sv.x0, Ly.peg.w, d, *dx_alt, c.pegT, c.pegH, c.pegW, D, Ly.peg.causal ? 2 : 1);
  PHK_LAUNCH_CHECK();
  *dx = *dx_alt;
  *dx_alt = d;
  return 0;
}

LayerCall step_layer_call(const Step& S) {
  LayerCall c;
  c.T = S.T; c.GT = S.GT; c.b = S.b; c.n = S.n;
  c.pegB = S.b; c.pegT = S.pt; c.pegH = S.ph; c.pegW = S.pw;
  c.bias = S.bias; c.dbias = S.dbias; c.key_mask = S.video_mask;
  c.context = S.context; c.L = S.L; c.text_mask = S.text_mask;
  c.prec = S.prec; c.s = S.s; c.st = S.st; c.tc = S.tc; c.asc = S.asc;
  return c;
}

// Stage 1.  wide_head: the bf16 operand buffers must hold the V-wide operands of the logits head.
int step_forward(Step& S, bool wide_head) {
  const phk_maskgit_t* m = S.m;
  const phk_transformer_t* T = S.T;
  const int b = S.b, n = S.n, pt = S.pt, ph = S.ph, pw = S.pw, L = S.L;
  const int D = S.D, H = S.H, DH = S.DH;
  const int64_t R = S.R, CR = S.CR;
  const phk_stream_t s = S.s;
  const cudaStream_t st = S.st;
  Arena& ar = S.ar;
  TcScratch& tc = S.tc;
  if (S.prec == PHK_PREC_BF16) {  // operand buffers of the wgmma products (activations stay fp32 everywhere else)
    tc.elems = tc_scratch_elems(m, R, CR, !wide_head);
    tc.a = reinterpret_cast<__nv_bfloat16*>(ar.f((tc.elems + 1) / 2));
    tc.b = reinterpret_cast<__nv_bfloat16*>(ar.f((tc.elems + 1) / 2));
    PHK_REQUIRE(tc.a && tc.b, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (tensor-core operands)");
  }

  float* x = ar.f(R * D);
  S.emb = ar.f(R * D);
  if (m->has_bias) {
    S.bias = ar.f((int64_t)H * n * n);
    S.dbias = ar.f((int64_t)H * n * n);
    float* sc = ar.f(phk_cpb_scratch_floats(&m->pos_bias, pt, ph, pw));
    PHK_REQUIRE(S.bias && S.dbias && sc, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (bias)");
    PHK_TRY(phk_cpb_bias(&m->pos_bias, pt, ph, pw, sc, S.bias, s));
    PHK_CUDA(cudaMemsetAsync(S.dbias, 0, (int64_t)H * n * n * 4, st));
  }
  PHK_REQUIRE(x && S.emb, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small");
  PHK_TRY(phk_token_embed(S.ids, m->token_emb, m->pos_emb, x, b, n, D, m->num_tokens + 1,
                          m->is_critic ? -1.f : m->shrink_alpha, 1, s));
  S.sv = new (std::nothrow) LayerSave[T->depth];
  PHK_REQUIRE(S.sv, PHK_E_ARG, "maskgit_train_step: out of host memory");
  if (S.drop_on) {
    S.bases = new (std::nothrow) uint64_t[T->depth][3];
    PHK_REQUIRE(S.bases, PHK_E_ARG, "maskgit_train_step: out of host memory");
    dropout_layout(m, b, n, S.context ? L : 0, S.bases);
  }
  // the attention backward's scratch; the forward's explicit attention path (dropout) uses it too
  const int nk_cross = L + 8;
  const int64_t as1 = attn_bwd_scratch_floats(b, H, n, n, DH), as2 = attn_bwd_scratch_floats(b, H, n, nk_cross, DH);
  S.asc = ar.f(as1 > as2 ? as1 : as2);
  PHK_REQUIRE(S.asc, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (attention scratch)");
  const LayerCall c = step_layer_call(S);
  const float* xin = x;
  for (int l = 0; l < T->depth; ++l) {
    PHK_REQUIRE(T->layers[l].has_peg, PHK_E_UNSUPPORTED, "maskgit_train_step: layers without PEG are not supported");
    float* xout = nullptr;
    PHK_TRY(layer_forward(c, l, xin, S.sv[l], &xout, ar, S.site(S.attn_p, l, 0), S.site(S.attn_p, l, 1), S.site(S.ff_p, l, 2)));
    xin = xout;
  }
  S.xf = xin;
  PHK_TRY(phk_layernorm(S.xf, T->out_g, T->out_b, S.emb, nullptr, R, D, 0, 0, 0, 0, s));
  return 0;
}

// The gradient buffers of stage 2 and 3: dxa / dxb (d/d residual stream), dtmp (d/d emb on entry to stage 3), stats.
int step_gradient_buffers(Step& S) {
  S.dxa = S.ar.f(S.R * S.D);
  S.dxb = S.ar.f(S.R * S.D);
  S.dtmp = S.ar.f(S.R * S.D);
  return S.dxa && S.dxb && S.dtmp ? 0 : -1;
}
int step_stats_buffer(Step& S) {
  S.stats = reinterpret_cast<float2*>(S.ar.f(2 * (S.R > S.CR ? S.R : S.CR)));
  return S.stats ? 0 : -1;
}

// Stage 3.  d_context (optional, [R_ctx, dim_context]): d/d(context) is ACCUMULATED into it over the cross-attention
// layers.  prog / nprog: the data-parallel progress events (phk_train_set_progress_events).
int step_backward(Step& S, float* d_context, void** prog, int nprog) {
  const phk_maskgit_t* m = S.m;
  const phk_maskgit_t* grads = S.grads;
  const phk_transformer_t* T = S.T;
  const phk_transformer_t* GT = S.GT;
  const int n = S.n, pt = S.pt, ph = S.ph, pw = S.pw;
  const int D = S.D, I = S.I;
  const int64_t R = S.R, CR = S.CR;
  const cudaStream_t st = S.st;
  const float* context = S.context;
  Arena& ar = S.ar;
  int64_t inner_max = 0, dc_max = 0;
  for (int l = 0; l < T->depth; ++l) {
    if (T->layers[l].ff.inner > inner_max) inner_max = T->layers[l].ff.inner;
    if (T->layers[l].has_cross && T->layers[l].cross_attn.dim_context > dc_max) dc_max = T->layers[l].cross_attn.dim_context;
  }
  LayerGrads G;
  G.dtmp = S.dtmp; G.stats = S.stats;
  G.dq = ar.f(R * I);
  G.dkv = ar.f(R * 2 * I);
  G.dob = ar.f(R * I);
  G.dh = ar.f(R * 2 * inner_max);
  G.dg = ar.f(R * inner_max);
  G.dckv = context ? ar.f(CR * 2 * I) : nullptr;
  G.dctxn = context ? ar.f(CR * (dc_max > 0 ? dc_max : 1)) : nullptr;
  PHK_REQUIRE(G.dq && G.dkv && G.dob && G.dh && G.dg && (!context || (G.dckv && G.dctxn)), PHK_E_WORKSPACE,
              "maskgit_train_step: workspace too small (gradients)");
  float* dx = S.dxa;      // d loss / d (current residual stream)
  float* dx_alt = S.dxb;
  PHK_TRY(ln_backward(S.xf, T->out_g, S.dtmp, dx, 0, (float*)GT->out_g, nullptr, S.stats, R, D, st));
  PHK_TRY(progress_mark(prog, nprog, 0, st));  // head + norm_out gradients final
  const LayerCall c = step_layer_call(S);
  for (int l = T->depth - 1; l >= 0; --l) {
    PHK_TRY(layer_backward(c, l, S.sv[l], &dx, &dx_alt, G, d_context, S.site(S.attn_p, l, 0), S.site(S.attn_p, l, 1),
                           S.site(S.ff_p, l, 2)));
    // this layer's parameter gradients are final -- except, with a context, the cross-attention's context_norm / to_kv
    // share nothing with other layers either; the position-bias gradient (dbias, all layers) is finished below
    PHK_TRY(progress_mark(prog, nprog, 1 + (T->depth - 1 - l), st));
  }
  // ---------------------------------------------------------------- embeddings, position-bias MLP
  const float alpha = m->is_critic ? 1.0f : m->shrink_alpha;
  if (t_det.p) {
    PHK_KERNEL_LAUNCH(embed_tok_fixed_kernel, dim3((unsigned)R), dim3(128), (size_t)(0), st, S.ids, (const float*)dx, (float*)grads->token_emb, R, D, alpha, m->num_tokens + 1);
    PHK_LAUNCH_CHECK();
    PHK_KERNEL_LAUNCH(embed_pos_fixed_kernel, dim3(ew_grid((int64_t)n * D)), dim3(256), (size_t)(0), st, (const float*)dx, (float*)grads->pos_emb, R, n, D, alpha);
    PHK_LAUNCH_CHECK();
  } else {
    PHK_KERNEL_LAUNCH(embed_bwd_kernel, dim3((unsigned)R), dim3(128), (size_t)(0), st, S.ids, dx, (float*)grads->token_emb, (float*)grads->pos_emb, n, D,
                                                 alpha, m->num_tokens + 1);
    PHK_LAUNCH_CHECK();
  }
  if (m->has_bias) {
    float* csc = ar.f(cpb_bwd_scratch_floats(m->pos_bias, pt, ph, pw));
    PHK_REQUIRE(csc, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (position-bias backward)");
    PHK_TRY(cpb_backward(m->pos_bias, grads->pos_bias, S.dbias, pt, ph, pw, csc, st));
  }
  PHK_TRY(progress_mark(prog, nprog, T->depth + 1, st));
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// Deterministic-mode scratch (t_det): the largest region any one reduction of the call uses, from the same per-site
// functions the reductions check against.  DetNeed keeps the maximum.
// ------------------------------------------------------------------------------------------------------------------
struct DetNeed {
  int64_t f = 0;
  void add(int64_t v) { f = v > f ? v : f; }
  void colsum(int64_t rows, int64_t cols) { add(colsum_fixed_floats(rows, cols)); }
  void ln(int64_t rows, int64_t dim) { add(ln_det_floats(rows, dim)); }
  void wgrad(int64_t M, int64_t N, int64_t K) { add(wgrad_det_floats(M, N, K)); }
};

// Every layer of T over b sequences of n rows (L > 0: cross-attention to L context tokens), and its norm_out
void det_need_stack(DetNeed& d, const phk_transformer_t* T, int b, int n, int L) {
  const int64_t R = (int64_t)b * n, CR = (int64_t)b * L, D = T->dim, I = (int64_t)T->heads * T->dim_head;
  d.ln(R, D);
  for (int l = 0; l < T->depth; ++l) {
    const phk_layer_t& Ly = T->layers[l];
    const int64_t inner = Ly.ff.inner;
    d.wgrad(R, D, inner); d.wgrad(R, 2 * inner, D); d.wgrad(R, D, I); d.wgrad(R, I, D); d.wgrad(R, 2 * I, D);
    d.add(attn_bwd_det_floats(AttnBwdGeom{b, T->heads, n, n, 0, T->dim_head}));
    if (Ly.has_peg) { d.colsum(R, D); d.add(peg_det_floats(D)); }
    if (Ly.has_cross && L > 0) {
      const int64_t dc = Ly.cross_attn.dim_context;
      d.ln(CR, dc); d.wgrad(CR, 2 * I, dc);
      d.add(attn_bwd_det_floats(AttnBwdGeom{b, T->heads, n, L, Ly.cross_attn.num_null_kv, T->dim_head}));
    }
  }
}

// cpb_backward over U coordinate deltas
void det_need_cpb(DetNeed& d, const phk_cpb_t& c, int64_t U) {
  d.wgrad(U, c.heads, c.hidden); d.wgrad(U, c.hidden, c.hidden); d.wgrad(U, c.hidden, c.num_dims);
  d.colsum(U, c.heads > c.hidden ? c.heads : c.hidden);
}

// stages 2 and 3 of a MaskGit differentiation of b sequences (head rows R = b n at most)
int64_t step_det_floats(const phk_maskgit_t* m, int32_t b, int32_t n, int32_t L) {
  DetNeed d;
  const int64_t R = (int64_t)b * n;
  det_need_stack(d, &m->transformer, b, n, L);
  d.colsum(R, m->num_tokens); d.wgrad(R, m->num_tokens, m->dim); d.wgrad(R, 1, m->dim);
  if (m->has_bias) det_need_cpb(d, m->pos_bias, 8 * (int64_t)n);  // U <= 8 n (step_workspace_bytes)
  return d.f;
}

// Bytes the deterministic mode adds to a workspace (0 in the default mode): the region and its alignment
int64_t det_bytes(int64_t floats) { return t_det_mode ? (floats > 0 ? floats : 1) * 4 + 256 : 0; }

// Carves the deterministic-mode region from the front of `ar` and publishes it for the call (nothing in the default mode)
int det_begin(Arena& ar, int64_t floats, const char* msg) {
  if (!t_det_mode) return 0;
  float* p = ar.f(floats > 0 ? floats : 1);
  PHK_REQUIRE(p, PHK_E_WORKSPACE, msg);
  t_det = DetScratch{p, floats};
  return 0;
}

// Workspace of one differentiation of b sequences: stage 1 and 3 (activations, gradient buffers, attention and
// position-bias scratch) + head_floats for stage 2; wide_head: the bf16 operand buffers hold the V-wide head operands.
int64_t step_workspace_bytes(const phk_maskgit_t* m, int32_t b, int32_t n, int32_t L, int64_t head_floats, bool wide_head,
                             int32_t prec) {
  const phk_transformer_t* T = &m->transformer;
  const int64_t R = (int64_t)b * n, CR = (int64_t)b * L, D = m->dim, I = (int64_t)T->heads * T->dim_head;
  int64_t inner = 0, dc = 0, f = 0;
  for (int l = 0; l < T->depth; ++l) {
    f += layer_save_floats(T, T->layers[l], R, CR);
    if (T->layers[l].ff.inner > inner) inner = T->layers[l].ff.inner;
    if (T->layers[l].has_cross && T->layers[l].cross_attn.dim_context > dc) dc = T->layers[l].cross_attn.dim_context;
  }
  f += R * D * 2;                                            // x (embedding output), final embeddings
  f += head_floats;
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
  if (prec == PHK_PREC_BF16) bytes += 2 * (tc_scratch_elems(m, R, CR, !wide_head) * 2 + 256);
  return bytes;
}

// widest dim_context of the cross-attention layers (0 without any)
int64_t context_width(const phk_transformer_t* T) {
  int64_t dc = 0;
  for (int l = 0; l < T->depth; ++l)
    if (T->layers[l].has_cross && T->layers[l].cross_attn.dim_context > dc) dc = T->layers[l].cross_attn.dim_context;
  return dc;
}

// set_error with the calling entry point's name in front ("entry: msg"), for the checks several entry points share
void set_entry_error(const char* entry, const char* msg) {
  char buf[256];
  std::snprintf(buf, sizeof(buf), "%s: %s", entry, msg);
  set_error(buf);
}
#define PHK_REQUIRE_IN(entry, cond, code, msg) \
  do { if (!(cond)) { set_entry_error(entry, msg); return (code); } } while (0)

// The argument and table checks of phk_maskgit_train_step and phk_maskgit_backward.  same_context_widths: every
// cross-attention layer must take contexts of one width (one buffer of the context serves them all).
int check_maskgit_call(const char* entry, const phk_maskgit_t* m, const phk_maskgit_t* grads, const int64_t* ids,
                       const void* workspace, int32_t b, int32_t n, int32_t pt, int32_t ph, int32_t pw, const float* context,
                       int32_t L, const uint8_t* text_mask, const float* d_context, int32_t prec, bool same_context_widths) {
  PHK_REQUIRE_IN(entry, m && grads && ids && workspace, PHK_E_ARG, "null pointer");
  PHK_REQUIRE_IN(entry, b > 0 && n > 0 && (int64_t)pt * ph * pw == n, PHK_E_SHAPE,
                 "video patch shape must cover the token sequence");
  PHK_REQUIRE_IN(entry, n <= m->max_seq_len, PHK_E_SHAPE,
                 "the video token sequence length is greater than max_seq_len (phenaki_pytorch.py:196)");
  PHK_REQUIRE_IN(entry, !context || (text_mask && L > 0), PHK_E_ARG, "context without text mask / length");
  PHK_REQUIRE_IN(entry, !d_context || context, PHK_E_ARG, "d_context without a context");
  PHK_REQUIRE_IN(entry, prec == PHK_PREC_F32 || prec == PHK_PREC_BF16, PHK_E_ARG, "unknown precision mode");
  const phk_transformer_t* T = &m->transformer;
  const phk_transformer_t* GT = &grads->transformer;
  PHK_REQUIRE_IN(entry, T->layers && GT->layers && T->depth > 0 && GT->depth == T->depth && !T->causal, PHK_E_ARG,
                 "transformer table / gradient table mismatch");
  PHK_REQUIRE_IN(entry, m->dim % 4 == 0, PHK_E_UNSUPPORTED, "dim must be a multiple of 4");
  if (same_context_widths) {
    const int64_t dc = context_width(T);
    for (int l = 0; l < T->depth; ++l)
      PHK_REQUIRE_IN(entry, !T->layers[l].has_cross || T->layers[l].cross_attn.dim_context == dc, PHK_E_UNSUPPORTED,
                     "cross-attention layers of different context widths");
  }
  return 0;
}

}  // namespace
}  // namespace phk

extern "C" int64_t phk_maskgit_train_workspace_bytes(const phk_maskgit_t* m, int32_t b, int32_t n, int32_t L,
                                                     int32_t bce_head, int32_t prec) {
  if (!m || b <= 0 || n <= 0 || L < 0 || !m->transformer.layers) return -1;
  const int64_t R = (int64_t)b * n;
  // (d)logits in place or the differentiated copy; row losses
  const int64_t head = bce_head ? 3 * R : R * (int64_t)m->num_tokens + 2 * R;
  return step_workspace_bytes(m, b, n, L, head, !bce_head, prec) + det_bytes(step_det_floats(m, b, n, L));
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
                                      int32_t prec, phk_stream_t s, const phk_dropout_t* dropout, float* d_context) {
  PHK_REQUIRE(loss_out, PHK_E_ARG, "maskgit_train_step: null pointer");
  // the context's gradient buffer serves every cross-attention layer
  PHK_TRY(check_maskgit_call("maskgit_train_step", m, grads, ids_in, workspace, b, n, pt, ph, pw, context, L, text_mask,
                             d_context, prec, d_context != nullptr));
  // head: labels given -> Linear(dim, 1) + BCE with logits (TokenCritic, or SelfCritic.to_pred on a MaskGit body,
  // phenaki_pytorch.py:307-336); otherwise to_logits + masked cross entropy
  const bool bce = labels != nullptr;
  PHK_REQUIRE(bce || (targets && token_mask), PHK_E_ARG,
              "maskgit_train_step: pass labels (critic head) or targets + token_mask (MaskGit head)");
  PHK_REQUIRE(bce || !m->is_critic, PHK_E_ARG, "maskgit_train_step: a TokenCritic table needs labels");
  PHK_REQUIRE(!(bce && logits_out), PHK_E_ARG, "maskgit_train_step: the critic head has no logits to hand back");
  PHK_REQUIRE(!d_context || (const float*)d_context != context, PHK_E_ARG, "maskgit_train_step: d_context aliases context");
  PHK_REQUIRE(workspace_bytes >= phk_maskgit_train_workspace_bytes(m, b, n, L, bce ? 1 : 0, prec), PHK_E_WORKSPACE,
              "maskgit_train_step: workspace too small");
  PHK_REQUIRE(!dropout || (dropout->attn_p >= 0.f && dropout->attn_p <= 1.f && dropout->ff_p >= 0.f && dropout->ff_p <= 1.f),
              PHK_E_ARG, "maskgit_train_step: dropout probabilities must lie in [0, 1]");
  void** prog = g_progress_events;  // one-shot: consumed by this call
  const int nprog = g_progress_count;
  g_progress_events = nullptr; g_progress_count = 0;
  Step S;
  S.m = m; S.grads = grads; S.ids = ids_in; S.b = b; S.n = n; S.pt = pt; S.ph = ph; S.pw = pw; S.L = L;
  S.context = context; S.text_mask = text_mask; S.video_mask = video_mask; S.prec = prec; S.s = s; S.dropout = dropout;
  S.ar = Arena{(char*)workspace, workspace_bytes, 0};
  DetScope det_scope;
  PHK_TRY(det_begin(S.ar, step_det_floats(m, b, n, L), "maskgit_train_step: workspace too small (deterministic mode)"));
  step_init(S);
  const cudaStream_t st = S.st;
  const int D = S.D, V = m->num_tokens;
  const int64_t R = S.R;

  // ---------------------------------------------------------------- forward (saving activations)
  PHK_TRY(step_forward(S, !bce));

  // ---------------------------------------------------------------- head + loss -> demb
  Arena& ar = S.ar;
  const int gb = step_gradient_buffers(S);
  float* row_loss = ar.f(R);
  float* cnt = ar.f(64);
  const int sb = step_stats_buffer(S);
  PHK_REQUIRE(gb == 0 && row_loss && cnt && sb == 0, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (bwd)");
  if (bce) {
    float* dscore = ar.f(R);
    PHK_REQUIRE(dscore, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small");
    PHK_KERNEL_LAUNCH(bce_rows_kernel, dim3((unsigned)((R + 7) / 8)), dim3(256), (size_t)(0), st, S.emb, m->head_w, m->head_b, labels, loss_scale, row_loss, dscore, R, D);
    PHK_LAUNCH_CHECK();
    PHK_TRY(wgrad(dscore, S.emb, (float*)grads->head_w, R, 1, D, st));  // [1, dim]: not worth a tensor-core launch
    PHK_TRY(colsum(dscore, R, 1, 1, (float*)grads->head_b, st));
    PHK_KERNEL_LAUNCH(outer_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, dscore, m->head_w, S.dtmp, R, D);
    PHK_LAUNCH_CHECK();
  } else {
    float* logits = logits_out ? logits_out : ar.f(R * (int64_t)V);
    PHK_REQUIRE(logits, PHK_E_WORKSPACE, "maskgit_train_step: workspace too small (logits)");
    PHK_TRY(linear_fwd(prec, S.tc, S.emb, m->head_w, logits, R, V, D, m->head_b, nullptr, s));
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
    PHK_TRY(wgrad_p(prec, S.tc, dl, S.emb, (float*)grads->head_w, R, V, D, s));
    PHK_TRY(colsum(dl, R, V, V, (float*)grads->head_b, st));
    PHK_TRY(dgrad_p(prec, S.tc, dl, m->head_w, S.dtmp, R, V, D, 0, s));
  }
  PHK_KERNEL_LAUNCH(loss_reduce_kernel, dim3(1), dim3(1024), (size_t)(0), st, row_loss, R, loss_out);
  PHK_LAUNCH_CHECK();

  // ---------------------------------------------------------------- backward through the transformer
  // (d_context: the context_norm backward each cross-attention layer runs for its gamma gradient also accumulates dx)
  return step_backward(S, d_context, prog, nprog);
}

// ------------------------------------------------------------------------------------------------------------------
// Backward from a caller-supplied gradient (include/phk.h, phk_maskgit_backward): stage 1 recomputes the forward of
// the module call being differentiated, stage 2 starts from the upstream gradient instead of a loss.
// Classifier-free-guidance pair: the forward ran 2b sequences, the second half under an all-false text mask, and
// returned out = null + s (cond - null).  The head is linear, so with g = d/d(out):
//   dW_head = g^T . (s E_cond + (1 - s) E_null),  db = colsum(g),  dE_cond = s (g . W),  dE_null = (1 - s) (g . W)
// -- one wgrad against the mixed embeddings and one dgrad, never a [2 b n, V] gradient.
// ------------------------------------------------------------------------------------------------------------------
namespace phk {
namespace {

// out = s a + (1 - s) b
__global__ void cfg_mix_kernel(const float* __restrict__ a, const float* __restrict__ b, float s, float* __restrict__ out,
                               int64_t total) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = s * a[i] + (1.0f - s) * b[i];
}
// d[half + i] = (1 - s) d[i], then d[i] = s d[i]: the gradient of both halves from that of the combined output
__global__ void cfg_split_kernel(float* __restrict__ d, float s, int64_t half) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = d[i];
    d[half + i] = (1.0f - s) * v;
    d[i] = s * v;
  }
}
// out[i] += a[i] + a[half + i]: the context gradient of both halves into the caller's
__global__ void add_halves_kernel(const float* __restrict__ a, float* __restrict__ out, int64_t half) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (int64_t)gridDim.x * blockDim.x)
    out[i] += a[i] + a[half + i];
}

// pair inputs of the CFG recompute: ids, video mask and context twice, the text mask then zeros
int64_t pair_input_floats(int64_t R, int64_t CR, int64_t dc) {
  return 2 * R * 2 + (2 * R + 3) / 4 + (2 * CR + 3) / 4 + 2 * CR * dc + 4 * 64;
}

}  // namespace
}  // namespace phk

extern "C" int64_t phk_maskgit_backward_workspace_bytes(const phk_maskgit_t* m, int32_t b, int32_t n, int32_t L,
                                                        int32_t cfg_pair, int32_t head_kind, int32_t prec) {
  if (!m || b <= 0 || n <= 0 || L < 0 || !m->transformer.layers) return -1;
  if (head_kind != PHK_HEAD_LOGITS && head_kind != PHK_HEAD_EMBEDS && head_kind != PHK_HEAD_SCORE) return -1;
  const bool pair = cfg_pair && L > 0;
  const int32_t B = pair ? 2 * b : b;
  const int64_t Rh = (int64_t)b * n, CRh = (int64_t)b * L, dc = context_width(&m->transformer);
  int64_t head = 64;
  if (pair) head += Rh * m->dim + pair_input_floats(Rh, CRh, dc) + 2 * CRh * dc;  // mixed embeddings; inputs; d context
  return step_workspace_bytes(m, B, n, L, head, head_kind == PHK_HEAD_LOGITS, prec) + det_bytes(step_det_floats(m, B, n, L));
}

// See include/phk.h.
extern "C" int phk_maskgit_backward(const phk_maskgit_t* m, const phk_maskgit_t* grads, const int64_t* ids, int32_t b,
                                    int32_t n, int32_t pt, int32_t ph, int32_t pw, const float* context, int32_t L,
                                    const uint8_t* text_mask, const uint8_t* video_mask, int32_t cfg_pair,
                                    float cond_scale, int32_t head_kind, const float* upstream, float* d_context,
                                    void* workspace, int64_t workspace_bytes, int32_t prec, phk_stream_t s) {
  PHK_REQUIRE(upstream, PHK_E_ARG, "maskgit_backward: null pointer");
  // the pair's copy of the context serves every cross-attention layer
  PHK_TRY(check_maskgit_call("maskgit_backward", m, grads, ids, workspace, b, n, pt, ph, pw, context, L, text_mask,
                             d_context, prec, context != nullptr));
  PHK_REQUIRE(head_kind == PHK_HEAD_LOGITS || head_kind == PHK_HEAD_EMBEDS || head_kind == PHK_HEAD_SCORE, PHK_E_ARG,
              "maskgit_backward: unknown head kind");
  PHK_REQUIRE(head_kind != PHK_HEAD_LOGITS || !m->is_critic, PHK_E_ARG, "maskgit_backward: a TokenCritic has no logits head");
  if (!context) L = 0;
  PHK_REQUIRE(workspace_bytes >= phk_maskgit_backward_workspace_bytes(m, b, n, L, cfg_pair, head_kind, prec), PHK_E_WORKSPACE,
              "maskgit_backward: workspace too small");
  const int64_t dc = context_width(&m->transformer);
  // without a context both halves of a pair are the same function of the weights: out = cond, no pair to differentiate
  const bool pair = cfg_pair && context;
  const float sc = pair ? cond_scale : 1.0f;
  cudaStream_t st = to_stream(s);
  const int64_t Rh = (int64_t)b * n, CRh = (int64_t)b * L;
  Step S;
  S.m = m; S.grads = grads; S.ids = ids; S.b = pair ? 2 * b : b; S.n = n; S.pt = pt; S.ph = ph; S.pw = pw; S.L = L;
  S.context = context; S.text_mask = text_mask; S.video_mask = video_mask; S.prec = prec; S.s = s;
  S.ar = Arena{(char*)workspace, workspace_bytes, 0};
  Arena& ar = S.ar;
  DetScope det_scope;
  PHK_TRY(det_begin(ar, step_det_floats(m, S.b, n, L), "maskgit_backward: workspace too small (deterministic mode)"));
  float* ctx_grad = d_context;  // where stage 3 accumulates d/d(context): both halves of a pair, summed below
  if (pair) {  // the 2b-sequence inputs of the forward's pair (phk_maskgit_forward, cfg_pair = 1)
    int64_t* ids2 = reinterpret_cast<int64_t*>(ar.f(2 * Rh * 2));
    uint8_t* vm2 = video_mask ? reinterpret_cast<uint8_t*>(ar.f((2 * Rh + 3) / 4)) : nullptr;
    uint8_t* tm2 = reinterpret_cast<uint8_t*>(ar.f((2 * CRh + 3) / 4));
    float* ctx2 = ar.f(2 * CRh * dc);
    PHK_REQUIRE(ids2 && (!video_mask || vm2) && tm2 && ctx2, PHK_E_WORKSPACE, "maskgit_backward: workspace too small (pair)");
    for (int h = 0; h < 2; ++h) {
      PHK_CUDA(cudaMemcpyAsync(ids2 + h * Rh, ids, Rh * 8, cudaMemcpyDeviceToDevice, st));
      if (video_mask) PHK_CUDA(cudaMemcpyAsync(vm2 + h * Rh, video_mask, Rh, cudaMemcpyDeviceToDevice, st));
      PHK_CUDA(cudaMemcpyAsync(ctx2 + h * CRh * dc, context, CRh * dc * 4, cudaMemcpyDeviceToDevice, st));
    }
    PHK_CUDA(cudaMemcpyAsync(tm2, text_mask, CRh, cudaMemcpyDeviceToDevice, st));
    PHK_CUDA(cudaMemsetAsync(tm2 + CRh, 0, CRh, st));  // the null half: every text token masked out
    S.ids = ids2; S.video_mask = vm2; S.text_mask = tm2; S.context = ctx2;
    if (d_context) {
      ctx_grad = ar.f(2 * CRh * dc);
      PHK_REQUIRE(ctx_grad, PHK_E_WORKSPACE, "maskgit_backward: workspace too small (context gradient)");
      PHK_CUDA(cudaMemsetAsync(ctx_grad, 0, 2 * CRh * dc * 4, st));
    }
  }
  step_init(S);
  const int D = S.D, V = m->num_tokens;

  // ---------------------------------------------------------------- stage 1: the forward, saving activations
  PHK_TRY(step_forward(S, head_kind == PHK_HEAD_LOGITS));

  // ---------------------------------------------------------------- stage 2: upstream gradient -> d emb
  PHK_REQUIRE(step_gradient_buffers(S) == 0 && step_stats_buffer(S) == 0, PHK_E_WORKSPACE,
              "maskgit_backward: workspace too small (bwd)");
  const float* emb_head = S.emb;  // what the head multiplied: the embeddings, or the pair's mix of both halves
  if (pair && head_kind != PHK_HEAD_EMBEDS) {
    float* mix = ar.f(Rh * D);
    PHK_REQUIRE(mix, PHK_E_WORKSPACE, "maskgit_backward: workspace too small (mixed embeddings)");
    PHK_KERNEL_LAUNCH(cfg_mix_kernel, dim3(ew_grid(Rh * D)), dim3(256), (size_t)(0), st, S.emb, S.emb + Rh * D, sc, mix, Rh * D);
    PHK_LAUNCH_CHECK();
    emb_head = mix;
  }
  if (head_kind == PHK_HEAD_LOGITS) {  // dlogits [b n, V]
    PHK_TRY(wgrad_p(prec, S.tc, upstream, emb_head, (float*)grads->head_w, Rh, V, D, s));
    PHK_TRY(colsum(upstream, Rh, V, V, (float*)grads->head_b, st));
    PHK_TRY(dgrad_p(prec, S.tc, upstream, m->head_w, S.dtmp, Rh, V, D, 0, s));
  } else if (head_kind == PHK_HEAD_SCORE) {  // dscore [b n]: the BCE head's branch of the train step without the BCE
    PHK_TRY(wgrad(upstream, emb_head, (float*)grads->head_w, Rh, 1, D, st));
    PHK_TRY(colsum(upstream, Rh, 1, 1, (float*)grads->head_b, st));
    PHK_KERNEL_LAUNCH(outer_kernel, dim3(ew_grid(Rh * D)), dim3(256), (size_t)(0), st, upstream, m->head_w, S.dtmp, Rh, D);
    PHK_LAUNCH_CHECK();
  } else {  // demb [b n, dim]: straight into the norm_out backward
    PHK_CUDA(cudaMemcpyAsync(S.dtmp, upstream, Rh * D * 4, cudaMemcpyDeviceToDevice, st));
  }
  if (pair) {
    PHK_KERNEL_LAUNCH(cfg_split_kernel, dim3(ew_grid(Rh * D)), dim3(256), (size_t)(0), st, S.dtmp, sc, Rh * D);
    PHK_LAUNCH_CHECK();
  }

  // ---------------------------------------------------------------- stage 3: transformer and embedding backward
  PHK_TRY(step_backward(S, ctx_grad, nullptr, 0));
  if (pair && d_context) {
    PHK_KERNEL_LAUNCH(add_halves_kernel, dim3(ew_grid(CRh * dc)), dim3(256), (size_t)(0), st, ctx_grad, d_context, CRh * dc);
    PHK_LAUNCH_CHECK();
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// C-ViViT decoder backward (include/phk.h, phk_cvivit_decode_backward): what autograd computes through CViViT.decode /
// decode_from_codebook_indices (cvivit.py:437-443, 476-516).  The forward is recomputed with saved activations on the
// layer code above, then differentiated from d video:
//   temporal stack  rows permuted from (b t h w) to (b h w t) by one gather, so that its sequences are runs of T' rows and
//                   the reference's raw x.reshape(b, t, h, w, d) of the (b h w, t, d) tensor (attention.py:71, the
//                   forward's peg_layout 1) is layout-0 PEG on these rows; ALiBi and the causal fill are one constant
//                   [H, T', T'] bias (-FLT_MAX above the diagonal: exact zeros in the softmax and in its backward)
//   spatial stack   rows (b t h w), runs of h w rows, no PEG; the 2-D continuous position bias sends its gradient through
//                   the bias MLP (cpb_backward with (h, w, 1))
//   to_pixels       norm_out gathered into first-frame / remaining-frame rows as the forward does; d video gathered into
//                   the same patch layout (the adjoint of phk_unpatchify); wgrad, bias column sum, dgrad per Linear
//   project_out     (ids) wgrad against the +-1 codes rebuilt from the ids and the bias column sum; the ids get nothing
// No dropout: the decode forward applies none.  phk_cvivit_backward runs the same decoder phase from d recon, then LFQ
// and the encoder's stacks and patch embeddings (DESIGN.md section 7.3).
// ------------------------------------------------------------------------------------------------------------------
namespace phk {
namespace {

// [B * Tp * hw, D] rows in (b, t, s) order -> (b, s, t) order (to_seq), or back
__global__ void permute_bts_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int Tp, int hw, int D,
                                   int to_seq) {
  const int64_t total = (int64_t)B * Tp * hw * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / D;
    const int d = (int)(i - r * D);
    int64_t sr;
    if (to_seq) {  // r = (b hw + s) Tp + t
      const int t = (int)(r % Tp);
      const int64_t bs = r / Tp;
      sr = ((bs / hw) * Tp + t) * hw + bs % hw;
    } else {       // r = (b Tp + t) hw + s
      const int s = (int)(r % hw);
      const int64_t bt = r / hw;
      sr = ((bt / Tp) * hw + s) * Tp + bt % Tp;
    }
    dst[i] = src[sr * D + d];
  }
}

// bias[h, i, j] = -|j - i| * slope[h] for j <= i, -FLT_MAX for j > i: ALiBi (attention.py:195-227) and the causal fill
// (:170-172) of the temporal attention, with the forward kernel's arithmetic (attention.cu)
__global__ void alibi_causal_bias_kernel(const float* __restrict__ slopes, float* __restrict__ bias, int H, int n) {
  const int64_t total = (int64_t)H * n * n;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx % n), i = (int)((idx / n) % n), h = (int)(idx / ((int64_t)n * n));
    bias[idx] = j > i ? -FLT_MAX : -fabsf((float)(j - i)) * slopes[h];
  }
}

// full[(b Tp + t) hw + s] = first[b hw + s] (t = 0) or rest[(b (Tp - 1) + t - 1) hw + s] (t > 0), rows of D floats
__global__ void frames_merge_kernel(const float* __restrict__ first, const float* __restrict__ rest, float* __restrict__ full,
                                    int B, int Tp, int hw, int D) {
  const int64_t total = (int64_t)B * Tp * hw * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / D;
    const int d = (int)(i - r * D);
    const int s = (int)(r % hw);
    const int t = (int)((r / hw) % Tp);
    const int64_t b = r / ((int64_t)hw * Tp);
    full[i] = t == 0 ? first[(b * hw + s) * D + d] : rest[((b * (Tp - 1) + t - 1) * hw + s) * D + d];
  }
}

// out[((b nt + t) hh + y) ww + x, ((c pt + k) p1 + i) p2 + j] = video[b, c, f0 + t pt + k, y p1 + i, x p2 + j]:
// 'b c (t pt) (h p1) (w p2) -> (b t h w) (c pt p1 p2)', the adjoint of phk_unpatchify (cvivit.py:286-295)
__global__ void patch_gather_kernel(const float* __restrict__ video, float* __restrict__ out, int B, int C, int F, int H,
                                    int W, int f0, int nt, int pt, int p1, int p2) {
  const int hh = H / p1, ww = W / p2, K = C * pt * p1 * p2;
  const int64_t total = (int64_t)B * nt * hh * ww * K;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / K;
    const int e = (int)(i - r * K);
    const int x = (int)(r % ww), y = (int)((r / ww) % hh), t = (int)((r / ((int64_t)ww * hh)) % nt);
    const int64_t b = r / ((int64_t)ww * hh * nt);
    const int j = e % p2, ii = (e / p2) % p1, k = (e / (p2 * p1)) % pt, c = e / (p2 * p1 * pt);
    out[i] = video[(((b * C + c) * F + f0 + (int64_t)t * pt + k) * H + (int64_t)y * p1 + ii) * W + (int64_t)x * p2 + j];
  }
}

// codes[r, k] = +1 if bit (bits - 1 - k) of ids[r] is set, else -1 (indices_to_codes before project_out, oracle/lfq.py)
__global__ void lfq_signs_kernel(const int64_t* __restrict__ ids, float* __restrict__ codes, int64_t rows, int bits) {
  const int64_t total = rows * bits;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / bits;
    const int k = (int)(i - r * bits);
    codes[i] = ((ids[r] >> (bits - 1 - k)) & 1) ? 1.0f : -1.0f;
  }
}

// video[b, c, f0 + t pt + k, y p1 + i, x p2 + j] += rows[((b nt + t) hh + y) ww + x, ((c pt + k) p1 + i) p2 + j]: the
// adjoint of patch_gather_kernel.  Patches tile the frames they cover, so every video element gets at most one term.
__global__ void patch_scatter_add_kernel(const float* __restrict__ rows, float* __restrict__ video, int B, int C, int F,
                                         int H, int W, int f0, int nt, int pt, int p1, int p2) {
  const int hh = H / p1, ww = W / p2, K = C * pt * p1 * p2;
  const int64_t total = (int64_t)B * nt * hh * ww * K;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / K;
    const int e = (int)(i - r * K);
    const int x = (int)(r % ww), y = (int)((r / ww) % hh), t = (int)((r / ((int64_t)ww * hh)) % nt);
    const int64_t b = r / ((int64_t)ww * hh * nt);
    const int j = e % p2, ii = (e / p2) % p1, k = (e / (p2 * p1)) % pt, c = e / (p2 * p1 * pt);
    video[(((b * C + c) * F + f0 + (int64_t)t * pt + k) * H + (int64_t)y * p1 + ii) * W + (int64_t)x * p2 + j] += rows[i];
  }
}

// first[b hw + s] = full[(b Tp) hw + s], rest[(b (Tp - 1) + t - 1) hw + s] = full[(b Tp + t) hw + s] (t > 0), rows of D
// floats: the adjoint of frames_merge_kernel
__global__ void frames_split_kernel(const float* __restrict__ full, float* __restrict__ first, float* __restrict__ rest,
                                    int B, int Tp, int hw, int D) {
  const int64_t total = (int64_t)B * Tp * hw * D;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / D;
    const int d = (int)(i - r * D);
    const int s = (int)(r % hw);
    const int t = (int)((r / hw) % Tp);
    const int64_t b = r / ((int64_t)hw * Tp);
    if (t == 0) first[(b * hw + s) * D + d] = full[i];
    else rest[((b * (Tp - 1) + t - 1) * hw + s) * D + d] = full[i];
  }
}

// Number of (B, F) frames a frame mask selects (NULL: all of them), counted by one thread in a fixed order
__device__ int64_t selected_frames(const uint8_t* __restrict__ mask, int B, int F) {
  if (!mask) return (int64_t)B * F;
  int64_t n = 0;
  for (int i = 0; i < B * F; ++i) n += mask[i] != 0;
  return n;
}

// Reconstruction loss (cvivit.py:584-590) over a (B, C, F, H, W) video: per-block fp64 partial sums of the masked squared
// error over a fixed grid, then one block adds the partials in a fixed order.  No atomics: two calls give bit-identical
// losses.
constexpr int kLossBlocks = PHK_RECON_LOSS_SCRATCH_BYTES / 8;

__global__ void __launch_bounds__(256) recon_loss_partial_kernel(const float* __restrict__ video,
                                                                 const float* __restrict__ recon,
                                                                 const uint8_t* __restrict__ mask, int C, int F,
                                                                 int64_t frame_elems, int64_t total,
                                                                 double* __restrict__ partial) {
  __shared__ double red[256];
  double a = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (mask) {
      const int64_t fr = i / frame_elems;  // ((b C + c) F + f)
      if (!mask[(fr / ((int64_t)C * F)) * F + fr % F]) continue;
    }
    const float d = recon[i] - video[i];
    a += (double)d * d;
  }
  red[threadIdx.x] = a;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(256) recon_loss_final_kernel(const double* __restrict__ partial,
                                                               const uint8_t* __restrict__ mask, int B, int C, int F,
                                                               int64_t frame_elems, float* __restrict__ loss) {
  __shared__ double red[256];
  double a = 0.0;
  for (int i = threadIdx.x; i < kLossBlocks; i += blockDim.x) a += partial[i];
  red[threadIdx.x] = a;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  // an all-false mask gives 0 / 0 = NaN, as the reference's mean over an empty selection does
  if (threadIdx.x == 0) *loss = (float)(red[0] / ((double)selected_frames(mask, B, F) * C * frame_elems));
}

// d recon = dloss 2 / N mask (recon - video) (+ the caller's d recon); d video = -(the same MSE term) (NULL: not wanted).
// N = selected frames C H W; with nothing selected the MSE term is zero (the reference's mean over an empty selection
// sends no gradient).
__global__ void __launch_bounds__(256) recon_grad_kernel(const float* __restrict__ video, const float* __restrict__ recon,
                                                         const uint8_t* __restrict__ mask, const float* __restrict__ dloss,
                                                         const float* __restrict__ drecon_in, float* __restrict__ drecon,
                                                         float* __restrict__ dvideo, int B, int C, int F,
                                                         int64_t frame_elems) {
  __shared__ float scale;
  if (threadIdx.x == 0) {
    const int64_t n = selected_frames(mask, B, F);
    scale = n > 0 ? (float)(2.0 * (double)*dloss / ((double)n * C * frame_elems)) : 0.f;
  }
  __syncthreads();
  const int64_t total = (int64_t)B * C * F * frame_elems;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    bool on = true;
    if (mask) {
      const int64_t fr = i / frame_elems;
      on = mask[(fr / ((int64_t)C * F)) * F + fr % F] != 0;
    }
    const float g = on ? scale * (recon[i] - video[i]) : 0.f;
    drecon[i] = drecon_in ? g + drecon_in[i] : g;
    if (dvideo) dvideo[i] = -g;
  }
}

int64_t stack_inner(const phk_transformer_t* T) {
  int64_t inner = 0;
  for (int l = 0; l < T->depth; ++l) inner = T->layers[l].ff.inner > inner ? T->layers[l].ff.inner : inner;
  return inner;
}

int64_t imax(int64_t a, int64_t b) { return a > b ? a : b; }

// Shapes of one C-ViViT backward: B videos of T' latent frames of hh x ww patches; R = B T' hh ww token rows;
// rows1 / rows2 = the first-frame / remaining-frame rows; K1 / K2 = their patch widths; inner = the widest FF
struct CvGeom {
  int B = 0, Tp = 0, hh = 0, ww = 0, hw = 0, D = 0, H = 0, DH = 0, I = 0, C = 0, F = 0;
  int64_t R = 0, rows1 = 0, rows2 = 0, K1 = 0, K2 = 0, inner = 0;
};

template <class M>  // phk_cvivit_t or phk_cvivit_dec_t: both carry the geometry fields read here
CvGeom cv_geom(const M* m, int B, int Tp, int64_t inner) {
  CvGeom g;
  g.B = B; g.Tp = Tp; g.hh = m->image_h / m->patch_h; g.ww = m->image_w / m->patch_w; g.hw = g.hh * g.ww;
  g.D = m->dim; g.H = m->heads; g.DH = m->dim_head; g.I = g.H * g.DH; g.C = m->channels; g.F = 1 + (Tp - 1) * m->patch_t;
  g.R = (int64_t)B * Tp * g.hw; g.rows1 = (int64_t)B * g.hw; g.rows2 = (int64_t)B * (Tp - 1) * g.hw;
  g.K1 = (int64_t)g.C * m->patch_h * m->patch_w; g.K2 = g.K1 * m->patch_t; g.inner = inner;
  return g;
}

// one bf16 operand buffer of the C-ViViT backward's tensor-core products (see tc_scratch_elems): every [rows, width]
// operand, straight or transposed, with width up to K2 = C pt p1 p2 (to_pixels / to_patch_emb)
int64_t cv_tc_scratch_elems(const CvGeom& g) {
  const int64_t width = imax(imax(2 * g.inner, 2 * (int64_t)g.I), imax(g.D, g.K2));
  const int64_t feat = imax(imax(g.D, g.I), g.inner);
  const int64_t tokens = pad8(g.R) + 8;
  return imax(tokens, feat + 8) * (width + 8);
}

// Buffers of a C-ViViT backward that every phase uses: the tensor-core operand scratch, the constant attention biases,
// the spatial position bias and its gradient (accumulated by every spatial stack), the attention and position-bias
// scratch, the two gradient streams dx / dx_alt and the layers' gradient scratch
struct CvShared {
  TcScratch tc{nullptr, nullptr, 0};
  float *bias_t = nullptr, *bias_s = nullptr, *dbias_s = nullptr, *cpb_sc = nullptr, *cpb_bwd_sc = nullptr, *asc = nullptr;
  float *dx = nullptr, *dx_alt = nullptr;
  LayerGrads G{};
};

int64_t cv_shared_floats(const CvGeom& g, const phk_cpb_t& cpb) {
  const int64_t a1 = attn_bwd_scratch_floats(g.B * g.hw, g.H, g.Tp, g.Tp, g.DH);
  const int64_t a2 = attn_bwd_scratch_floats(g.B * g.Tp, g.H, g.hw, g.hw, g.DH);
  int64_t f = (int64_t)g.H * g.Tp * g.Tp + 2 * (int64_t)g.H * g.hw * g.hw;       // biases, d spatial bias
  f += phk_cpb_scratch_floats(&cpb, g.hh, g.ww, 1) + cpb_bwd_scratch_floats(cpb, g.hh, g.ww, 1) + imax(a1, a2);
  f += 2 * g.R * g.D;                                                             // dx, dx_alt
  f += g.R * (g.D + 4 * (int64_t)g.I + 3 * g.inner) + 2 * g.R;                    // dtmp | dq dkv(2) dob | dh(2) dg | stats
  return f;
}
int64_t cv_shared_bytes(const CvGeom& g, const phk_cpb_t& cpb, int prec) {
  int64_t bytes = cv_shared_floats(g, cpb) * 4 + 256 * 24;
  if (prec == PHK_PREC_BF16) bytes += 2 * (cv_tc_scratch_elems(g) * 2 + 256);
  return bytes;
}

// Takes the shared buffers from `ar`, computes the spatial position bias and zeroes its gradient.
int cv_shared_init(Arena& ar, const CvGeom& g, const phk_cpb_t& cpb, int prec, phk_stream_t s, CvShared& S) {
  if (prec == PHK_PREC_BF16) {
    S.tc.elems = cv_tc_scratch_elems(g);
    S.tc.a = reinterpret_cast<__nv_bfloat16*>(ar.f((S.tc.elems + 1) / 2));
    S.tc.b = reinterpret_cast<__nv_bfloat16*>(ar.f((S.tc.elems + 1) / 2));
    PHK_REQUIRE(S.tc.a && S.tc.b, PHK_E_WORKSPACE, "cvivit backward: workspace too small (tensor-core operands)");
  }
  const int64_t a1 = attn_bwd_scratch_floats(g.B * g.hw, g.H, g.Tp, g.Tp, g.DH);
  const int64_t a2 = attn_bwd_scratch_floats(g.B * g.Tp, g.H, g.hw, g.hw, g.DH);
  S.bias_t = ar.f((int64_t)g.H * g.Tp * g.Tp);
  S.bias_s = ar.f((int64_t)g.H * g.hw * g.hw);
  S.dbias_s = ar.f((int64_t)g.H * g.hw * g.hw);
  S.cpb_sc = ar.f(phk_cpb_scratch_floats(&cpb, g.hh, g.ww, 1));
  S.cpb_bwd_sc = ar.f(cpb_bwd_scratch_floats(cpb, g.hh, g.ww, 1));
  S.asc = ar.f(imax(a1, a2));
  S.dx = ar.f(g.R * g.D);
  S.dx_alt = ar.f(g.R * g.D);
  LayerGrads& G = S.G;
  G.dtmp = ar.f(g.R * g.D); G.dq = ar.f(g.R * g.I); G.dkv = ar.f(g.R * 2 * g.I); G.dob = ar.f(g.R * g.I);
  G.dh = ar.f(g.R * 2 * g.inner); G.dg = ar.f(g.R * g.inner); G.dckv = nullptr; G.dctxn = nullptr;
  G.stats = reinterpret_cast<float2*>(ar.f(2 * g.R));
  PHK_REQUIRE(S.bias_t && S.bias_s && S.dbias_s && S.cpb_sc && S.cpb_bwd_sc && S.asc && S.dx && S.dx_alt && G.dtmp && G.dq &&
              G.dkv && G.dob && G.dh && G.dg && G.stats, PHK_E_WORKSPACE, "cvivit backward: workspace too small");
  PHK_TRY(phk_cpb_bias(&cpb, g.hh, g.ww, 1, S.cpb_sc, S.bias_s, s));
  PHK_CUDA(cudaMemsetAsync(S.dbias_s, 0, (int64_t)g.H * g.hw * g.hw * 4, to_stream(s)));
  return 0;
}

// The temporal stack of C-ViViT (encoder or decoder) on (b h w t) rows: B h w sequences of T' rows, layout-0 PEG over
// (B, T', h, w) (the reference's raw reshape of these rows), ALiBi plus the causal fill as one constant bias, written
// into S.bias_t here
int temporal_call(const phk_transformer_t* T, const phk_transformer_t* GT, const CvGeom& g, const CvShared& S, int prec,
                  phk_stream_t s, LayerCall* c) {
  *c = LayerCall();
  c->T = T; c->GT = GT; c->b = g.B * g.hw; c->n = g.Tp;
  c->pegB = g.B; c->pegT = g.Tp; c->pegH = g.hh; c->pegW = g.ww;
  c->bias = S.bias_t; c->prec = prec; c->s = s; c->st = to_stream(s); c->tc = S.tc; c->asc = S.asc;
  PHK_KERNEL_LAUNCH(alibi_causal_bias_kernel, dim3(ew_grid((int64_t)g.H * g.Tp * g.Tp)), dim3(256), (size_t)(0), c->st, T->alibi_slopes, S.bias_t, g.H, g.Tp);
  PHK_LAUNCH_CHECK();
  return 0;
}

// The spatial stack on (b t h w) rows: B T' sequences of h w rows, no PEG, the 2-D position bias (its gradient
// accumulates into S.dbias_s)
LayerCall spatial_call(const phk_transformer_t* T, const phk_transformer_t* GT, const CvGeom& g, const CvShared& S,
                       int prec, phk_stream_t s) {
  LayerCall c;
  c.T = T; c.GT = GT; c.b = g.B * g.Tp; c.n = g.hw;
  c.pegB = g.B; c.pegT = g.Tp; c.pegH = g.hh; c.pegW = g.ww;
  c.bias = S.bias_s; c.dbias = S.dbias_s; c.prec = prec; c.s = s; c.st = to_stream(s); c.tc = S.tc; c.asc = S.asc;
  return c;
}

// Every layer of c.T on x (saving activations into sv[depth]); *xf = the stack's output before norm_out
int stack_forward(const LayerCall& c, const float* x, LayerSave* sv, const float** xf, Arena& ar) {
  const DropSite none{0.f, 0.f, 0u, 0u, 0u};
  for (int l = 0; l < c.T->depth; ++l) {
    float* xout = nullptr;
    PHK_TRY(layer_forward(c, l, x, sv[l], &xout, ar, none, none, none));
    x = xout;
  }
  *xf = x;
  return 0;
}

// Backward of norm_out(stack(x)) from dy = d/d(norm_out output): on return *dx holds d/d(x) (*dx, *dx_alt may swap).
// prog: one event per layer, top layer (with norm_out) first
int stack_backward(const LayerCall& c, const LayerSave* sv, const float* xf, const float* dy, float** dx, float** dx_alt,
                   const LayerGrads& G, Progress* prog) {
  const DropSite none{0.f, 0.f, 0u, 0u, 0u};
  const int64_t R = (int64_t)c.b * c.n;
  PHK_TRY(ln_backward(xf, c.T->out_g, dy, *dx, 0, (float*)c.GT->out_g, nullptr, G.stats, R, c.T->dim, c.st));
  for (int l = c.T->depth - 1; l >= 0; --l) {
    PHK_TRY(layer_backward(c, l, sv[l], dx, dx_alt, G, nullptr, none, none, none));
    PHK_TRY(progress_next(prog, c.st));
  }
  return 0;
}

int64_t dec_phase_floats(const phk_cvivit_dec_t* m, const CvGeom& g) {
  int64_t f = 2 * g.R * g.D;                                                     // codes (b t h w), their (b h w t) copy
  for (int l = 0; l < m->temporal.depth; ++l) f += layer_save_floats(&m->temporal, m->temporal.layers[l], g.R, 0);
  for (int l = 0; l < m->spatial.depth; ++l) f += layer_save_floats(&m->spatial, m->spatial.layers[l], g.R, 0);
  f += 2 * g.R * g.D;                                                            // temporal norm_out (b h w t), spatial input
  f += 2 * (g.rows1 + imax(g.rows2, 1)) * g.D;                                   // spatial norm_out and its gradient, split
  f += imax(g.rows1 * g.K1, g.rows2 * g.K2);                                     // d video in a patch layout
  f += g.R * imax(m->codebook_bits, 1);                                          // +-1 codes
  return f + 256 * 16 / 4;
}

// The decoder half of both backward entry points: recomputes the decode with its activations saved in `ar` (a copy: all
// of it is dead on return) and differentiates it from d video.  With ids, project_out's gradients are accumulated.
// cpb_now: finish the position-bias MLP's gradient here; otherwise S.dbias_s is left to the caller.  dcodes_out (or
// dtokens): receives d/d(decoder input) in (b t h w) rows, in dtokens when given, else in a free gradient stream of S.
// prog (NULL: none): one event after to_pixels*, one per spatial then temporal layer, one after project_out (ids only).
int decode_backward_phase(const phk_cvivit_dec_t* m, const phk_cvivit_dec_t* grads, const int64_t* ids, const float* tokens,
                          const CvGeom& g, const float* dvideo, float* dtokens, const float** dcodes_out, const CvShared& S,
                          Arena ar, bool cpb_now, int prec, phk_stream_t s, Progress* prog) {
  const phk_transformer_t* TT = &m->temporal;
  const phk_transformer_t* TS = &m->spatial;
  const int B = g.B, Tp = g.Tp, hw = g.hw, D = g.D, C = g.C, F = g.F;
  const int64_t R = g.R, per = (int64_t)Tp * hw, K1 = g.K1, K2 = g.K2, rows1 = g.rows1, rows2 = g.rows2;
  const cudaStream_t st = to_stream(s);
  float* xc = ar.f(R * D);
  float* xp = ar.f(R * D);
  PHK_REQUIRE(xc && xp, PHK_E_WORKSPACE, "cvivit_decode_backward: workspace too small");

  // ---------------------------------------------------------------- inputs
  const float* x_in = tokens;
  if (ids) {
    PHK_TRY(phk_lfq_codes(ids, m->vq_out_w, m->vq_out_b, xc, R, D, m->codebook_bits, s));
    x_in = xc;
  }
  PHK_KERNEL_LAUNCH(permute_bts_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, x_in, xp, B, Tp, hw, D, 1);
  PHK_LAUNCH_CHECK();

  // ---------------------------------------------------------------- forward, saving activations
  LayerCall ct;
  PHK_TRY(temporal_call(TT, &grads->temporal, g, S, prec, s, &ct));
  const LayerCall cs = spatial_call(TS, &grads->spatial, g, S, prec, s);
  std::unique_ptr<LayerSave[]> svT(new (std::nothrow) LayerSave[TT->depth]), svS(new (std::nothrow) LayerSave[TS->depth]);
  PHK_REQUIRE(svT && svS, PHK_E_ARG, "cvivit_decode_backward: out of host memory");
  const float* xfT = nullptr;
  PHK_TRY(stack_forward(ct, xp, svT.get(), &xfT, ar));
  float* nT = ar.f(R * D);
  float* P = ar.f(R * D);
  PHK_REQUIRE(nT && P, PHK_E_WORKSPACE, "cvivit_decode_backward: workspace too small");
  PHK_TRY(phk_layernorm(xfT, TT->out_g, TT->out_b, nT, nullptr, R, D, 0, 0, 0, 0, s));
  PHK_KERNEL_LAUNCH(permute_bts_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, nT, P, B, Tp, hw, D, 0);
  PHK_LAUNCH_CHECK();
  const float* xfS = nullptr;
  PHK_TRY(stack_forward(cs, P, svS.get(), &xfS, ar));
  float* Ef = ar.f(rows1 * D);
  float* Er = ar.f((rows2 > 0 ? rows2 : 1) * D);
  PHK_REQUIRE(Ef && Er, PHK_E_WORKSPACE, "cvivit_decode_backward: workspace too small");
  PHK_TRY(phk_layernorm(xfS, TS->out_g, TS->out_b, Ef, nullptr, rows1, D, 0, -hw, per, 0, s));
  if (Tp > 1) PHK_TRY(phk_layernorm(xfS, TS->out_g, TS->out_b, Er, nullptr, rows2, D, 0, -(per - hw), per, hw, s));

  // ---------------------------------------------------------------- to_pixels_first_frame / to_pixels
  const LayerGrads& G = S.G;
  float* dx = S.dx;
  float* dx_alt = S.dx_alt;
  float* dG = ar.f(imax(rows1 * K1, rows2 * K2));
  float* dEf = ar.f(rows1 * D);
  float* dEr = ar.f((rows2 > 0 ? rows2 : 1) * D);
  PHK_REQUIRE(dG && dEf && dEr, PHK_E_WORKSPACE, "cvivit_decode_backward: workspace too small (gradients)");
  PHK_KERNEL_LAUNCH(patch_gather_kernel, dim3(ew_grid(rows1 * K1)), dim3(256), (size_t)(0), st, dvideo, dG, B, C, F, m->image_h, m->image_w, 0, 1, 1, m->patch_h, m->patch_w);
  PHK_LAUNCH_CHECK();
  PHK_TRY(wgrad_p(prec, S.tc, dG, Ef, (float*)grads->px_first_w, rows1, K1, D, s));
  PHK_TRY(colsum(dG, rows1, (int)K1, K1, (float*)grads->px_first_b, st));
  PHK_TRY(dgrad_p(prec, S.tc, dG, m->px_first_w, dEf, rows1, K1, D, 0, s));
  if (Tp > 1) {  // (one latent frame: to_pixels sees an empty batch, its gradients stay the caller's zeros)
    PHK_KERNEL_LAUNCH(patch_gather_kernel, dim3(ew_grid(rows2 * K2)), dim3(256), (size_t)(0), st, dvideo, dG, B, C, F, m->image_h, m->image_w, 1, Tp - 1, m->patch_t, m->patch_h, m->patch_w);
    PHK_LAUNCH_CHECK();
    PHK_TRY(wgrad_p(prec, S.tc, dG, Er, (float*)grads->px_w, rows2, K2, D, s));
    PHK_TRY(colsum(dG, rows2, (int)K2, K2, (float*)grads->px_b, st));
    PHK_TRY(dgrad_p(prec, S.tc, dG, m->px_w, dEr, rows2, K2, D, 0, s));
  }
  PHK_TRY(progress_next(prog, st));  // to_pixels_first_frame / to_pixels final
  PHK_KERNEL_LAUNCH(frames_merge_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, dEf, dEr, G.dtmp, B, Tp, hw, D);
  PHK_LAUNCH_CHECK();

  // ---------------------------------------------------------------- spatial stack, position-bias MLP
  PHK_TRY(stack_backward(cs, svS.get(), xfS, G.dtmp, &dx, &dx_alt, G, prog));
  if (cpb_now) PHK_TRY(cpb_backward(m->spatial_bias, grads->spatial_bias, S.dbias_s, g.hh, g.ww, 1, S.cpb_bwd_sc, st));

  // ---------------------------------------------------------------- temporal stack, rows (b h w t)
  PHK_KERNEL_LAUNCH(permute_bts_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, dx, G.dtmp, B, Tp, hw, D, 1);
  PHK_LAUNCH_CHECK();
  PHK_TRY(stack_backward(ct, svT.get(), xfT, G.dtmp, &dx, &dx_alt, G, prog));

  // ---------------------------------------------------------------- d tokens / project_out
  if (!ids && !dtokens && !dcodes_out) return 0;
  float* dcodes = dtokens ? dtokens : dx_alt;
  PHK_KERNEL_LAUNCH(permute_bts_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, dx, dcodes, B, Tp, hw, D, 0);
  PHK_LAUNCH_CHECK();
  if (dcodes_out) *dcodes_out = dcodes;
  if (ids) {
    const int bits = m->codebook_bits;
    float* signs = ar.f(R * bits);
    PHK_REQUIRE(signs, PHK_E_WORKSPACE, "cvivit_decode_backward: workspace too small (codes)");
    PHK_KERNEL_LAUNCH(lfq_signs_kernel, dim3(ew_grid(R * bits)), dim3(256), (size_t)(0), st, ids, signs, R, bits);
    PHK_LAUNCH_CHECK();
    PHK_TRY(wgrad(dcodes, signs, (float*)grads->vq_out_w, R, D, bits, st));  // [dim, bits]: not worth a tensor-core launch
    PHK_TRY(colsum(dcodes, R, D, D, (float*)grads->vq_out_b, st));
    PHK_TRY(progress_next(prog, st));  // project_out final
  }
  return 0;
}

// Arena space of encode_backward_phase: the layers' saves, the spatial norm_out, its (b h w t) copy, the temporal norm_out
int64_t enc_stacks_floats(const phk_cvivit_t* m, const CvGeom& g) {
  int64_t f = 3 * g.R * g.D;
  for (int l = 0; l < m->spatial.depth; ++l) f += layer_save_floats(&m->spatial, m->spatial.layers[l], g.R, 0);
  for (int l = 0; l < m->temporal.depth; ++l) f += layer_save_floats(&m->temporal, m->temporal.layers[l], g.R, 0);
  return f + 256 * 4 / 4;
}

// Arena space of phk_cvivit_backward's encoder phase (the stacks' space is dead before the patch gradients are taken,
// but it is counted in full)
int64_t enc_phase_floats(const phk_cvivit_t* m, const CvGeom& g, bool dvideo) {
  const int64_t rows2 = imax(g.rows2, 1);
  const int64_t patch = imax(g.rows1 * g.K1, g.rows2 * g.K2);
  int64_t f = 2 * (g.rows1 * g.K1 + rows2 * g.K2);                               // raw patch rows, LN1 outputs
  f += (g.rows1 + rows2) * g.D + 2 * g.R * g.D;                                  // Linear outputs, LN2 outputs, z (b t h w)
  f += enc_stacks_floats(m, g);
  f += (g.rows1 + rows2) * g.D + imax(g.rows1, rows2) * g.D;                     // d LN2 outputs split, d Linear outputs
  f += patch * (dvideo ? 2 : 1);                                                 // d LN1 outputs, d patch rows
  return f + 256 * 16 / 4;
}

// The encoder stacks' half of both encoder backward entry points (cvivit.py:449-474): recomputes the spatial stack on x0
// ((b t h w) rows) and the temporal stack on its permuted norm_out with their activations saved in `ar` (a copy: all of it
// is dead on return), then differentiates norm_out(temporal) from dout ((b t h w) rows; it may be one of S's gradient
// streams).  z (NULL: not formed): receives the recomputed output, (b t h w) rows.  On return *dx0 = d x0 in (b t h w)
// rows, in a gradient stream of S; dtokens (NULL: not wanted) receives a copy (written, not added).  cpb_now: finish the
// position-bias MLP's gradient here; otherwise S.dbias_s is left to the caller.  prog (NULL: none): one event per
// temporal then spatial layer.
int encode_backward_phase(const phk_cvivit_t* m, const phk_cvivit_t* grads, const float* x0, const CvGeom& g,
                          const float* dout, float* z, float* dtokens, const float** dx0, const CvShared& S, Arena ar,
                          bool cpb_now, int prec, phk_stream_t s, Progress* prog) {
  const phk_transformer_t* ES = &m->spatial;
  const phk_transformer_t* ET = &m->temporal;
  const int B = g.B, Tp = g.Tp, hw = g.hw, D = g.D;
  const int64_t R = g.R;
  const cudaStream_t st = to_stream(s);

  // ---------------------------------------------------------------- forward, saving activations
  const LayerCall cs = spatial_call(ES, &grads->spatial, g, S, prec, s);
  LayerCall ct;
  PHK_TRY(temporal_call(ET, &grads->temporal, g, S, prec, s, &ct));
  std::unique_ptr<LayerSave[]> svS(new (std::nothrow) LayerSave[ES->depth]), svT(new (std::nothrow) LayerSave[ET->depth]);
  PHK_REQUIRE(svT && svS, PHK_E_ARG, "cvivit_encode_backward: out of host memory");
  const float* xfS = nullptr;
  PHK_TRY(stack_forward(cs, x0, svS.get(), &xfS, ar));
  float* nS = ar.f(R * D); float* Pt = ar.f(R * D);
  PHK_REQUIRE(nS && Pt, PHK_E_WORKSPACE, "cvivit_encode_backward: workspace too small");
  PHK_TRY(phk_layernorm(xfS, ES->out_g, ES->out_b, nS, nullptr, R, D, 0, 0, 0, 0, s));
  PHK_KERNEL_LAUNCH(permute_bts_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, nS, Pt, B, Tp, hw, D, 1);
  PHK_LAUNCH_CHECK();
  const float* xfT = nullptr;
  PHK_TRY(stack_forward(ct, Pt, svT.get(), &xfT, ar));
  if (z) {
    float* nT = ar.f(R * D);
    PHK_REQUIRE(nT, PHK_E_WORKSPACE, "cvivit_encode_backward: workspace too small");
    PHK_TRY(phk_layernorm(xfT, ET->out_g, ET->out_b, nT, nullptr, R, D, 0, 0, 0, 0, s));
    PHK_KERNEL_LAUNCH(permute_bts_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, nT, z, B, Tp, hw, D, 0);
    PHK_LAUNCH_CHECK();
  }

  // ---------------------------------------------------------------- temporal stack on (b h w t) rows, then spatial
  const LayerGrads& G = S.G;
  float* dx = S.dx;
  float* dx_alt = S.dx_alt;
  PHK_KERNEL_LAUNCH(permute_bts_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, dout, G.dtmp, B, Tp, hw, D, 1);
  PHK_LAUNCH_CHECK();
  PHK_TRY(stack_backward(ct, svT.get(), xfT, G.dtmp, &dx, &dx_alt, G, prog));
  PHK_KERNEL_LAUNCH(permute_bts_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, dx, G.dtmp, B, Tp, hw, D, 0);
  PHK_LAUNCH_CHECK();
  PHK_TRY(stack_backward(cs, svS.get(), xfS, G.dtmp, &dx, &dx_alt, G, prog));
  if (dtokens) PHK_CUDA(cudaMemcpyAsync(dtokens, dx, R * D * 4, cudaMemcpyDeviceToDevice, st));
  if (dx0) *dx0 = dx;
  if (cpb_now) PHK_TRY(cpb_backward(m->spatial_bias, grads->spatial_bias, S.dbias_s, g.hh, g.ww, 1, S.cpb_bwd_sc, st));
  return 0;
}

template <class M>  // phk_cvivit_t or phk_cvivit_dec_t
bool cvivit_shapes_ok(const M* m, int32_t B, int32_t Tp) {
  return m && B > 0 && Tp > 0 && m->temporal.layers && m->spatial.layers && m->temporal.depth > 0 && m->spatial.depth > 0 &&
         m->patch_h > 0 && m->patch_w > 0 && m->patch_t > 0 && m->image_h % m->patch_h == 0 && m->image_w % m->patch_w == 0;
}

// The checks of one side's weight table against its gradient table that every C-ViViT backward makes: the stacks'
// depths and widths, the temporal stack causal with ALiBi slopes and the spatial one not, no cross-attention layer.
template <class M>  // phk_cvivit_t or phk_cvivit_dec_t
int check_cvivit_pair(const char* entry, const M* m, const M* grads) {
  const phk_transformer_t* TT = &m->temporal;
  const phk_transformer_t* TS = &m->spatial;
  PHK_REQUIRE_IN(entry, grads->temporal.layers && grads->spatial.layers && grads->temporal.depth == TT->depth &&
                 grads->spatial.depth == TS->depth, PHK_E_ARG, "weight table / gradient table mismatch");
  PHK_REQUIRE_IN(entry, TT->causal && TT->alibi_slopes && !TS->causal, PHK_E_ARG,
                 "the temporal stack is causal with ALiBi slopes, the spatial one is not");
  PHK_REQUIRE_IN(entry, TT->dim == m->dim && TS->dim == m->dim && TT->heads == m->heads && TS->heads == m->heads &&
                 TT->dim_head == m->dim_head && TS->dim_head == m->dim_head, PHK_E_ARG,
                 "transformer widths differ from the model's");
  PHK_REQUIRE_IN(entry, m->dim % 4 == 0, PHK_E_UNSUPPORTED, "dim must be a multiple of 4");
  const phk_transformer_t* stacks[2] = {TT, TS};
  for (const phk_transformer_t* T : stacks)
    for (int l = 0; l < T->depth; ++l) PHK_REQUIRE_IN(entry, !T->layers[l].has_cross, PHK_E_ARG, "cross-attention layer");
  return 0;
}

// Deterministic-mode scratch (see step_det_floats) of the C-ViViT backward phases
void det_need_cv_stacks(DetNeed& d, const phk_transformer_t* TT, const phk_transformer_t* TS, const CvGeom& g) {
  det_need_stack(d, TT, g.B * g.hw, g.Tp, 0);
  det_need_stack(d, TS, g.B * g.Tp, g.hw, 0);
}
void det_need_cv_cpb(DetNeed& d, const phk_cpb_t& c, const CvGeom& g) {
  det_need_cpb(d, c, (int64_t)(2 * g.hh - 1) * (2 * g.ww - 1));
}
int64_t cv_decode_det_floats(const phk_cvivit_dec_t* m, const CvGeom& g) {
  DetNeed d;
  det_need_cv_stacks(d, &m->temporal, &m->spatial, g);
  d.wgrad(g.rows1, g.K1, g.D); d.colsum(g.rows1, g.K1); d.wgrad(g.rows2, g.K2, g.D); d.colsum(g.rows2, g.K2);  // to_pixels*
  d.wgrad(g.R, g.D, m->codebook_bits); d.colsum(g.R, g.D);                                                    // project_out
  det_need_cv_cpb(d, m->spatial_bias, g);
  return d.f;
}
int64_t cv_encode_det_floats(const phk_cvivit_t* m, const CvGeom& g) {
  DetNeed d;
  det_need_cv_stacks(d, &m->temporal, &m->spatial, g);
  det_need_cv_cpb(d, m->spatial_bias, g);
  return d.f;
}
int64_t cv_backward_det_floats(const phk_cvivit_t* enc, const phk_cvivit_dec_t* dec, const CvGeom& g) {
  DetNeed d;
  d.add(cv_decode_det_floats(dec, g));
  d.add(cv_encode_det_floats(enc, g));
  d.wgrad(g.R, enc->codebook_bits, g.D); d.colsum(g.R, enc->codebook_bits);  // project_in
  const int64_t rows[2] = {g.rows1, g.rows2}, K[2] = {g.K1, g.K2};
  for (int e = 0; e < 2; ++e) {  // to_patch_emb*: LN -> Linear -> LN
    d.ln(rows[e], g.D); d.wgrad(rows[e], g.D, K[e]); d.colsum(rows[e], g.D); d.ln(rows[e], K[e]);
  }
  return d.f;
}

}  // namespace
}  // namespace phk

extern "C" int64_t phk_cvivit_decode_backward_workspace_bytes(const phk_cvivit_dec_t* m, int32_t B, int32_t Tp, int32_t prec) {
  if (!cvivit_shapes_ok(m, B, Tp)) return -1;
  const CvGeom g = cv_geom(m, B, Tp, imax(stack_inner(&m->temporal), stack_inner(&m->spatial)));
  return cv_shared_bytes(g, m->spatial_bias, prec) + dec_phase_floats(m, g) * 4 + det_bytes(cv_decode_det_floats(m, g));
}

// See include/phk.h.
extern "C" int phk_cvivit_decode_backward(const phk_cvivit_dec_t* m, const phk_cvivit_dec_t* grads, const int64_t* ids,
                                          const float* tokens, int32_t B, int32_t Tp, const float* dvideo, float* dtokens,
                                          void* workspace, int64_t workspace_bytes, int32_t prec, phk_stream_t s) {
  PHK_REQUIRE(m && grads && (ids || tokens) && dvideo && workspace, PHK_E_ARG, "cvivit_decode_backward: null pointer");
  PHK_REQUIRE(!ids || !dtokens, PHK_E_ARG, "cvivit_decode_backward: dtokens belongs to the float-token decode (ids NULL)");
  PHK_REQUIRE(prec == PHK_PREC_F32 || prec == PHK_PREC_BF16, PHK_E_ARG, "cvivit_decode_backward: unknown precision mode");
  const int64_t need = phk_cvivit_decode_backward_workspace_bytes(m, B, Tp, prec);
  PHK_REQUIRE(need > 0, PHK_E_ARG, "cvivit_decode_backward: bad model table or shape");
  PHK_REQUIRE(workspace_bytes >= need, PHK_E_WORKSPACE, "cvivit_decode_backward: workspace too small");
  PHK_TRY(check_cvivit_pair("cvivit_decode_backward", m, grads));
  PHK_REQUIRE(!ids || (m->codebook_bits > 0 && m->vq_out_w && m->vq_out_b && grads->vq_out_w && grads->vq_out_b), PHK_E_ARG,
              "cvivit_decode_backward: ids need LFQ's project_out and its gradient");
  const CvGeom g = cv_geom(m, B, Tp, imax(stack_inner(&m->temporal), stack_inner(&m->spatial)));
  Arena ar{(char*)workspace, workspace_bytes, 0};
  DetScope det_scope;
  PHK_TRY(det_begin(ar, cv_decode_det_floats(m, g), "cvivit_decode_backward: workspace too small (deterministic mode)"));
  CvShared S;
  PHK_TRY(cv_shared_init(ar, g, m->spatial_bias, prec, s, S));
  return decode_backward_phase(m, grads, ids, tokens, g, dvideo, dtokens, nullptr, S, ar, true, prec, s, nullptr);
}

// See include/phk.h.
extern "C" int phk_cvivit_recon_loss(const float* video, const float* recon, const uint8_t* frame_mask, int32_t B,
                                     int32_t C, int32_t F, int32_t H, int32_t W, void* scratch, float* loss_out,
                                     phk_stream_t s) {
  PHK_REQUIRE(video && recon && scratch && loss_out, PHK_E_ARG, "cvivit_recon_loss: null pointer");
  PHK_REQUIRE(B > 0 && C > 0 && F > 0 && H > 0 && W > 0, PHK_E_ARG, "cvivit_recon_loss: bad size");
  const cudaStream_t st = to_stream(s);
  const int64_t frame = (int64_t)H * W, total = (int64_t)B * C * F * frame;
  double* partial = reinterpret_cast<double*>(scratch);
  PHK_KERNEL_LAUNCH(recon_loss_partial_kernel, dim3(kLossBlocks), dim3(256), (size_t)(0), st, video, recon, frame_mask, C, F, frame, total, partial);
  PHK_LAUNCH_CHECK();
  PHK_KERNEL_LAUNCH(recon_loss_final_kernel, dim3(1), dim3(256), (size_t)(0), st, (const double*)partial, frame_mask, B, C, F, frame, loss_out);
  PHK_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t phk_cvivit_backward_workspace_bytes(const phk_cvivit_t* enc, const phk_cvivit_dec_t* dec, int32_t B,
                                                       int32_t F, int32_t prec) {
  if (!enc || !dec || F <= 0 || dec->patch_t <= 0 || (F - 1) % dec->patch_t != 0) return -1;
  const int Tp = 1 + (F - 1) / dec->patch_t;
  if (!cvivit_shapes_ok(dec, B, Tp) || !enc->spatial.layers || !enc->temporal.layers || enc->spatial.depth <= 0 ||
      enc->temporal.depth <= 0 || enc->codebook_bits <= 0)
    return -1;
  const int64_t inner = imax(imax(stack_inner(&dec->temporal), stack_inner(&dec->spatial)),
                             imax(stack_inner(&enc->temporal), stack_inner(&enc->spatial)));
  const CvGeom g = cv_geom(dec, B, Tp, inner);
  const int64_t video = (int64_t)B * g.C * F * dec->image_h * dec->image_w;
  const int64_t own = g.R * enc->codebook_bits + video + 256 * 4 / 4;            // d q, d recon
  return cv_shared_bytes(g, dec->spatial_bias, prec) + (own + imax(dec_phase_floats(dec, g), enc_phase_floats(enc, g, true))) * 4 +
         det_bytes(cv_backward_det_floats(enc, dec, g));
}

// See include/phk.h: to_pixels*, the decoder's spatial and temporal layers, project_out, the encoder's temporal and
// spatial layers, project_in, to_patch_emb*, the position-bias MLP.
extern "C" int32_t phk_cvivit_backward_progress_groups(const phk_cvivit_t* enc, const phk_cvivit_dec_t* dec) {
  if (!enc || !dec || enc->spatial.depth <= 0 || enc->temporal.depth <= 0 || dec->spatial.depth <= 0 ||
      dec->temporal.depth <= 0)
    return -1;
  return 1 + dec->spatial.depth + dec->temporal.depth + 1 + enc->temporal.depth + enc->spatial.depth + 1 + 1 + 1;
}

// See include/phk.h.  Order: d recon; the decoder phase (as phk_cvivit_decode_backward, from the forward's ids); LFQ
// (project_out's dgrad, the straight-through d x = d q, project_in); the encoder phase (recomputed with saved activations
// in the space the decoder phase used, then differentiated down to the patch rows and d video); the position-bias MLP
// once, over the bias gradient both spatial stacks accumulated.
extern "C" int phk_cvivit_backward(const phk_cvivit_t* enc, const phk_cvivit_t* enc_grads, const phk_cvivit_dec_t* dec,
                                   const phk_cvivit_dec_t* dec_grads, const float* video, const float* recon,
                                   const int64_t* ids, const uint8_t* frame_mask, int32_t B, int32_t F, const float* dloss,
                                   const float* drecon, float* dvideo, int32_t straight_through, void* workspace,
                                   int64_t workspace_bytes, int32_t prec, phk_stream_t s) {
  Progress prog{g_progress_events, g_progress_count, 0};  // one-shot: consumed by this call, even one that fails
  g_progress_events = nullptr; g_progress_count = 0;
  PHK_REQUIRE(enc && enc_grads && dec && dec_grads && video && recon && ids && dloss && workspace, PHK_E_ARG,
              "cvivit_backward: null pointer");
  PHK_REQUIRE(prec == PHK_PREC_F32 || prec == PHK_PREC_BF16, PHK_E_ARG, "cvivit_backward: unknown precision mode");
  const int64_t need = phk_cvivit_backward_workspace_bytes(enc, dec, B, F, prec);
  PHK_REQUIRE(need > 0, PHK_E_ARG, "cvivit_backward: bad model table or shape (LFQ tokenizers only)");
  PHK_REQUIRE(workspace_bytes >= need, PHK_E_WORKSPACE, "cvivit_backward: workspace too small");
  PHK_REQUIRE(enc->dim == dec->dim && enc->heads == dec->heads && enc->dim_head == dec->dim_head &&
              enc->channels == dec->channels && enc->image_h == dec->image_h && enc->image_w == dec->image_w &&
              enc->patch_h == dec->patch_h && enc->patch_w == dec->patch_w && enc->patch_t == dec->patch_t &&
              enc->codebook_bits == dec->codebook_bits, PHK_E_ARG, "cvivit_backward: encoder and decoder tables differ in shape");
  PHK_REQUIRE(enc->vq_w && enc->vq_b && enc_grads->vq_w && enc_grads->vq_b && dec->vq_out_w && dec->vq_out_b &&
              dec_grads->vq_out_w && dec_grads->vq_out_b, PHK_E_ARG, "cvivit_backward: LFQ's projections and their gradients");
  PHK_TRY(check_cvivit_pair("cvivit_backward", enc, enc_grads));
  PHK_TRY(check_cvivit_pair("cvivit_backward", dec, dec_grads));
  const phk_transformer_t* ES = &enc->spatial;
  const phk_transformer_t* ET = &enc->temporal;
  const int Tp = 1 + (F - 1) / dec->patch_t;
  const int64_t inner = imax(imax(stack_inner(&dec->temporal), stack_inner(&dec->spatial)), imax(stack_inner(ET), stack_inner(ES)));
  const CvGeom g = cv_geom(dec, B, Tp, inner);
  const int D = g.D, hw = g.hw, bits = enc->codebook_bits, C = g.C, H = dec->image_h, W = dec->image_w;
  const int64_t R = g.R, rows1 = g.rows1, rows2 = g.rows2, K1 = g.K1, K2 = g.K2;
  const int64_t nvideo = (int64_t)B * C * F * H * W;
  const cudaStream_t st = to_stream(s);
  Arena ar{(char*)workspace, workspace_bytes, 0};
  DetScope det_scope;
  PHK_TRY(det_begin(ar, cv_backward_det_floats(enc, dec, g), "cvivit_backward: workspace too small (deterministic mode)"));
  CvShared S;
  PHK_TRY(cv_shared_init(ar, g, dec->spatial_bias, prec, s, S));
  float* dq = ar.f(R * bits);
  float* drec = ar.f(nvideo);
  PHK_REQUIRE(dq && drec, PHK_E_WORKSPACE, "cvivit_backward: workspace too small");

  // ---------------------------------------------------------------- d recon (and the MSE term of d video)
  PHK_KERNEL_LAUNCH(recon_grad_kernel, dim3(ew_grid(nvideo)), dim3(256), (size_t)(0), st, video, recon, frame_mask, dloss, drecon, drec, dvideo, B, C, F, (int64_t)H * W);
  PHK_LAUNCH_CHECK();

  // ---------------------------------------------------------------- decoder phase, from the forward's ids
  const float* dcodes = nullptr;
  PHK_TRY(decode_backward_phase(dec, dec_grads, ids, nullptr, g, drec, nullptr, &dcodes, S, ar, false, prec, s, &prog));

  // ---------------------------------------------------------------- LFQ: d q = d z_dec W_out; straight through, d x = d q
  if (straight_through) {
    PHK_TRY(dgrad(dcodes, dec->vq_out_w, dq, R, D, bits, 0, st));  // [R, bits]: the LFQ products stay fp32 (bits wide)

    // ---------------------------------------------------------------- encoder phase: recompute
    Arena ea = ar;  // the decoder phase's space
    const int64_t r2 = rows2 > 0 ? rows2 : 1;
    float* X1 = ea.f(rows1 * K1); float* A1 = ea.f(rows1 * K1);
    float* X2 = ea.f(r2 * K2); float* A2 = ea.f(r2 * K2);
    float* Pe1 = ea.f(rows1 * D); float* Pe2 = ea.f(r2 * D);
    float* x0 = ea.f(R * D);
    PHK_REQUIRE(X1 && A1 && X2 && A2 && Pe1 && Pe2 && x0, PHK_E_WORKSPACE, "cvivit_backward: workspace too small (patches)");
    PHK_KERNEL_LAUNCH(patch_gather_kernel, dim3(ew_grid(rows1 * K1)), dim3(256), (size_t)(0), st, video, X1, B, C, F, H, W, 0, 1, 1, enc->patch_h, enc->patch_w);
    PHK_LAUNCH_CHECK();
    PHK_TRY(phk_patchify_ln(video, B, C, F, H, W, 0, 1, 1, enc->patch_h, enc->patch_w, enc->pf_ln1_g, enc->pf_ln1_b, A1, 0, s));
    PHK_TRY(linear_fwd(prec, S.tc, A1, enc->pf_w, Pe1, rows1, D, K1, enc->pf_b, nullptr, s));
    PHK_TRY(phk_layernorm(Pe1, enc->pf_ln2_g, enc->pf_ln2_b, x0, nullptr, rows1, D, 0, hw, (int64_t)Tp * hw, 0, s));
    if (rows2 > 0) {
      PHK_KERNEL_LAUNCH(patch_gather_kernel, dim3(ew_grid(rows2 * K2)), dim3(256), (size_t)(0), st, video, X2, B, C, F, H, W, 1, Tp - 1, enc->patch_t, enc->patch_h, enc->patch_w);
      PHK_LAUNCH_CHECK();
      PHK_TRY(phk_patchify_ln(video, B, C, F, H, W, 1, Tp - 1, enc->patch_t, enc->patch_h, enc->patch_w, enc->pr_ln1_g,
                              enc->pr_ln1_b, A2, 0, s));
      PHK_TRY(linear_fwd(prec, S.tc, A2, enc->pr_w, Pe2, rows2, D, K2, enc->pr_b, nullptr, s));
      PHK_TRY(phk_layernorm(Pe2, enc->pr_ln2_g, enc->pr_ln2_b, x0, nullptr, rows2, D, 0, (int64_t)(Tp - 1) * hw,
                            (int64_t)Tp * hw, hw, s));
    }
    float* z = ea.f(R * D);
    PHK_REQUIRE(z, PHK_E_WORKSPACE, "cvivit_backward: workspace too small");

    // ---------------------------------------------------------------- the two stacks, then project_in against their output
    const LayerGrads& G = S.G;
    PHK_TRY(dgrad(dq, enc->vq_w, S.dx, R, bits, D, 0, st));  // d(encoder output), (b t h w)
    const float* dx = nullptr;
    PHK_TRY(encode_backward_phase(enc, enc_grads, x0, g, S.dx, z, nullptr, &dx, S, ea, false, prec, s, &prog));
    PHK_TRY(wgrad(dq, z, (float*)enc_grads->vq_w, R, bits, D, st));
    PHK_TRY(colsum(dq, R, bits, bits, (float*)enc_grads->vq_b, st));
    PHK_TRY(progress_next(&prog, st));  // project_in final

    // ---------------------------------------------------------------- to_patch_emb_first_frame / to_patch_emb
    float* dE1 = ea.f(rows1 * D); float* dE2 = ea.f(r2 * D);
    float* dP = ea.f(imax(rows1, r2) * D);
    float* dA = ea.f(imax(rows1 * K1, rows2 * K2));
    float* dX = dvideo ? ea.f(imax(rows1 * K1, rows2 * K2)) : nullptr;
    PHK_REQUIRE(dE1 && dE2 && dP && dA && (dX || !dvideo), PHK_E_WORKSPACE, "cvivit_backward: workspace too small (patch gradients)");
    PHK_KERNEL_LAUNCH(frames_split_kernel, dim3(ew_grid(R * D)), dim3(256), (size_t)(0), st, dx, dE1, dE2, B, Tp, hw, D);
    PHK_LAUNCH_CHECK();
    struct Emb { const float *X, *A, *Pe, *dE, *ln1_g, *w, *ln2_g; const phk_cvivit_t* gr; int64_t rows, K; int f0, nt, pt; bool first; };
    const Emb embs[2] = {{X1, A1, Pe1, dE1, enc->pf_ln1_g, enc->pf_w, enc->pf_ln2_g, enc_grads, rows1, K1, 0, 1, 1, true},
                         {X2, A2, Pe2, dE2, enc->pr_ln1_g, enc->pr_w, enc->pr_ln2_g, enc_grads, rows2, K2, 1, Tp - 1, enc->patch_t, false}};
    for (const Emb& e : embs) {
      if (e.rows == 0) continue;  // (one latent frame: to_patch_emb sees an empty batch, its gradients stay zero)
      float* g_ln1_g = (float*)(e.first ? e.gr->pf_ln1_g : e.gr->pr_ln1_g);
      float* g_ln1_b = (float*)(e.first ? e.gr->pf_ln1_b : e.gr->pr_ln1_b);
      float* g_w = (float*)(e.first ? e.gr->pf_w : e.gr->pr_w);
      float* g_b = (float*)(e.first ? e.gr->pf_b : e.gr->pr_b);
      float* g_ln2_g = (float*)(e.first ? e.gr->pf_ln2_g : e.gr->pr_ln2_g);
      float* g_ln2_b = (float*)(e.first ? e.gr->pf_ln2_b : e.gr->pr_ln2_b);
      // nn.LayerNorm with a bias parameter: dbeta is a gradient here
      PHK_TRY(ln_backward(e.Pe, e.ln2_g, e.dE, dP, 0, g_ln2_g, g_ln2_b, G.stats, e.rows, D, st));
      PHK_TRY(wgrad_p(prec, S.tc, dP, e.A, g_w, e.rows, D, e.K, s));
      PHK_TRY(colsum(dP, e.rows, D, D, g_b, st));
      PHK_TRY(dgrad_p(prec, S.tc, dP, e.w, dA, e.rows, D, e.K, 0, s));
      PHK_TRY(ln_backward(e.X, e.ln1_g, dA, dX, 0, g_ln1_g, g_ln1_b, G.stats, e.rows, (int)e.K, st));
      if (dvideo) {
        PHK_KERNEL_LAUNCH(patch_scatter_add_kernel, dim3(ew_grid(e.rows * e.K)), dim3(256), (size_t)(0), st, (const float*)dX, dvideo, B, C, F, H, W, e.f0, e.nt, e.pt, enc->patch_h, enc->patch_w);
        PHK_LAUNCH_CHECK();
      }
    }
    PHK_TRY(progress_next(&prog, st));  // to_patch_emb_first_frame / to_patch_emb final
  } else {
    // eval mode: the encoder's groups are empty, their events are recorded all the same (the count depends on the tables only)
    for (int k = 0; k < ET->depth + ES->depth + 2; ++k) PHK_TRY(progress_next(&prog, st));
  }

  // ---------------------------------------------------------------- position-bias MLP, once over both spatial stacks
  PHK_TRY(cpb_backward(dec->spatial_bias, dec_grads->spatial_bias, S.dbias_s, g.hh, g.ww, 1, S.cpb_bwd_sc, st));
  return progress_next(&prog, st);  // the position-bias MLP final: every gradient is
}

extern "C" int64_t phk_cvivit_encode_backward_workspace_bytes(const phk_cvivit_t* m, int32_t B, int32_t Tp, int32_t prec) {
  if (!cvivit_shapes_ok(m, B, Tp)) return -1;
  const CvGeom g = cv_geom(m, B, Tp, imax(stack_inner(&m->spatial), stack_inner(&m->temporal)));
  return cv_shared_bytes(g, m->spatial_bias, prec) + enc_stacks_floats(m, g) * 4 + det_bytes(cv_encode_det_floats(m, g));
}

// See include/phk.h.
extern "C" int phk_cvivit_encode_backward(const phk_cvivit_t* m, const phk_cvivit_t* grads, const float* tokens, int32_t B,
                                          int32_t Tp, const float* dout, float* dtokens, void* workspace,
                                          int64_t workspace_bytes, int32_t prec, phk_stream_t s) {
  PHK_REQUIRE(m && grads && tokens && dout && workspace, PHK_E_ARG, "cvivit_encode_backward: null pointer");
  PHK_REQUIRE(prec == PHK_PREC_F32 || prec == PHK_PREC_BF16, PHK_E_ARG, "cvivit_encode_backward: unknown precision mode");
  const int64_t need = phk_cvivit_encode_backward_workspace_bytes(m, B, Tp, prec);
  PHK_REQUIRE(need > 0, PHK_E_ARG, "cvivit_encode_backward: bad model table or shape");
  PHK_REQUIRE(workspace_bytes >= need, PHK_E_WORKSPACE, "cvivit_encode_backward: workspace too small");
  PHK_TRY(check_cvivit_pair("cvivit_encode_backward", m, grads));
  const phk_cpb_t& gc = grads->spatial_bias;
  PHK_REQUIRE(gc.w0 && gc.b0 && gc.w1 && gc.b1 && gc.w2 && gc.b2, PHK_E_ARG,
              "cvivit_encode_backward: the gradient table has no position-bias MLP");
  const CvGeom g = cv_geom(m, B, Tp, imax(stack_inner(&m->spatial), stack_inner(&m->temporal)));
  Arena ar{(char*)workspace, workspace_bytes, 0};
  DetScope det_scope;
  PHK_TRY(det_begin(ar, cv_encode_det_floats(m, g), "cvivit_encode_backward: workspace too small (deterministic mode)"));
  CvShared S;
  PHK_TRY(cv_shared_init(ar, g, m->spatial_bias, prec, s, S));
  return encode_backward_phase(m, grads, tokens, g, dout, nullptr, dtokens, nullptr, S, ar, true, prec, s, nullptr);
}
