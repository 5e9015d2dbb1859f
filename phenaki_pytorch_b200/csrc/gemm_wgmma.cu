// bf16 GEMM on the Hopper tensor cores (sm_90a, wgmma):
//   C[map(m), n] = sum_k A[m,k] * W[n,k]  (+bias) (+residual)        nn.Linear semantics
// A, W bf16, K-major (row-major [rows, K]); fp32 accumulation in registers.
//
// gemm_bf16_kernel<EPI, DUAL> behind phk_gemm_bf16 / phk_gemm_bf16_x2 / _qkv / _qnorm: one CTA per 128 x 128 tile,
// DUAL = two independent problems in one persistent launch.  Persistent (one CTA per SM, static round-robin tile
// scheduler, m-fastest so concurrent CTAs share the W tile in L2 while the A panel stays L2-resident):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor.2d (SWIZZLE_128B) stages 128x64 A and W tiles into
//                   a 4-deep shared-memory ring; out-of-bounds rows / the K tail are zero-filled by the TMA unit.
//   warpgroups 1..4 each multiplies one 64 x 64 quadrant of the tile (wgmma.m64n64k16, both operands from shared
//                   memory), writes it into the epilogue's staging layout, and then all sixteen warps run the epilogue
//                   (four per 32-row group, each a quarter of the columns) while the producer fills the ring for the
//                   next tile.
// Epilogues: 0 fp32 (+bias, +residual, row map) -- through the TMA unit when the row map is the identity: the
//              residual tile is bulk-loaded into SWIZZLE_128B staging boxes during the main loop and the result tile
//              bulk-stored from them; otherwise staged in a padded smem tile and written with coalesced rows
//            1 bf16 (+bias)
//            2 GEGLU (attention.py:40-43) on W rows packed [64 value rows | 64 gate rows] per 128-column tile ->
//              bf16 [M, N/2]: fitted sigmoid-form GELU, swizzled bf16 staging tile, coalesced 16-byte stores.
#include "phk_common.cuh"
#include "phk_sm90.cuh"
#include <mutex>
#include <unordered_map>

namespace phk {

constexpr int GM = 128;       // BLOCK_M: two wgmma M = 64 halves
constexpr int GN = 128;       // BLOCK_N: two 64-column halves
constexpr int GK = 64;        // BLOCK_K: 64 bf16 = 128 B = one SWIZZLE_128B row
constexpr int GSTAGES = 4;
constexpr int EPI_WARPS = 16;       // MMA + epilogue warps 4..19: four per 32-row group, each a quarter of the columns
constexpr int EPI_PARTS = EPI_WARPS / 4;            // column parts per row group
constexpr int GTHREADS = 128 + EPI_WARPS * 32;      // 640: the producer warpgroup + four MMA / epilogue warpgroups
constexpr int STAGE_BYTES = GM * GK * 2;          // 16 KB per operand per stage
constexpr int CPAD = 132;                          // fp32 staging row stride (floats): conflict-free 128-bit rows
constexpr int CSTAGE_BYTES = GM * CPAD * 4;        // 67.6 KB
constexpr int RING_BYTES = GSTAGES * 2 * STAGE_BYTES;
constexpr int SMEM_TOTAL = RING_BYTES + CSTAGE_BYTES + 256 /*barriers*/ + 1024 /*manual 1024-B alignment*/;

struct EpiParams {
  void* C; int64_t ldc; int64_t M; int N; int K;
  const float* bias; const float* residual;
  int64_t seg_len, seg_stride, seg_off;
  int m_tiles, n_tiles;
  // fp32 epilogue through the TMA unit (identity row map, C 16-B aligned, residual == C or none): C as a tensor map
  // with [128 rows x 32 floats] SWIZZLE_128B boxes; the residual tile is bulk-LOADED into the staging boxes while the
  // main loop runs and the finished tile is bulk-STORED from them, so the epilogue warps issue no global accesses
  int tma_epi;
  // epilogue 3 (self-attention operands, attention.py:146-157): bf16 output; columns [0, norm_cols) are l2-normalised
  // per 64-column head (F.normalize, eps 1e-12), multiplied by nscale[col % 64] (q_scale / k_scale) and by nmul (the
  // fixed similarity scale 8 folded into q); columns >= norm_cols (the value half of to_kv) are only converted
  const float* nscale; int norm_cols; float nmul;
  alignas(64) CUtensorMap tmC;
};


__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(EPI_WARPS * 32) : "memory"); }

// One warpgroup's 64 x 64 accumulator quadrant (rows rq.., columns cq.. of the tile; warp w of the warpgroup) into the
// epilogue's staging layout, added onto the residual already staged there when `add` is set.  BOX: the four
// [128 rows x 128 B] SWIZZLE_128B boxes of the TMA epilogue; otherwise rows of CPAD floats.
template <bool BOX>
__device__ __forceinline__ void acc_to_stage(const float (&d)[32], uint8_t* stage, int rq, int cq, int w, int lane,
                                             bool add) {
  const int r0 = rq + 16 * w + (lane >> 2);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = cq + 8 * j + 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + 8 * h;
      float2* dst = BOX ? reinterpret_cast<float2*>(stage + (c >> 5) * (GM * 128) + r * 128 +
                                                    ((((c & 31) >> 2) ^ (r & 7)) << 4) + (c & 3) * 4)
                        : reinterpret_cast<float2*>(reinterpret_cast<float*>(stage) + r * CPAD + c);
      float2 v = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
      if (add) { const float2 o = *dst; v.x += o.x; v.y += o.y; }
      *dst = v;
    }
  }
}

// gelu_erf(g) * v for the bf16 GEGLU epilogue (attention.py:40-43).  Phi(g) = 0.5 (1 + erf(g / sqrt2)) is evaluated
// as sigmoid(2 g (a + b g^2 + c g^4)) with (a, b, c) fitted to the erf form (unlike 0.5 (1 + erf) from a polynomial, no
// cancellation for negative g), and sigmoid(z) = 0.5 + 0.5 tanh(z / 2) on ONE MUFU op (tanh.approx.f32, relative error
// 2^-11): a few issue slots per output instead of ~19 for the erf polynomial, because the epilogue is issue-bound.  Phi
// is good to 2.4e-4 absolute -- below the bf16 rounding of the hidden activations.  g^2 is clamped to 64: beyond |g| = 8
// the fitted quintic would turn over, while the sigmoid is already saturated.
__device__ __forceinline__ float geglu_fast(float g, float v) {
  const float g2 = fminf(g * g, 64.0f);
  float u = fmaf(g2, -0.00035151678851506f, 0.037005646021930225f);
  u = fmaf(u, g2, 0.7975078842858219f);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(g * u));
  const float h = 0.5f * (g * v);
  return fmaf(h, t, h);
}

// ---------------------------------------------------------------------------------------------------
// Epilogue pieces.  A "chunk" is the tile's 128 rows x 128 accumulator columns, staged in shared memory by
// acc_to_stage.
// ---------------------------------------------------------------------------------------------------

// Residual prefetch: while the main loop of the tile runs, pull the residual chunk into the staging buffer with
// coalesced 512-B row loads (the previous chunk's write-out finished at its closing barrier).
template <int EPI>
__device__ __forceinline__ bool epi_residual_prefetch(const EpiParams& p, float* cstage, int64_t m0, int n0, int ew,
                                                      int lane) {
  const bool res_vec = EPI == 0 && p.residual && (p.ldc % 4 == 0) && (p.N % 4 == 0) &&
                       ((reinterpret_cast<uintptr_t>(p.residual) & 15) == 0);
  if (res_vec) {
    const int col = n0 + lane * 4;
    const uint32_t seg_len = (uint32_t)p.seg_len;
#pragma unroll 1
    for (int rb = 0; rb < GM / EPI_WARPS; rb += 8) {
      float4 rv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int r = (rb + u) * EPI_WARPS + ew;
        const uint32_t m = (uint32_t)m0 + r;
        uint32_t orow = m;
        if (seg_len > 0) { const uint32_t q = m / seg_len; orow = q * (uint32_t)p.seg_stride + (uint32_t)p.seg_off + (m - q * seg_len); }
        rv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m < (uint32_t)p.M && col < p.N) rv[u] = *reinterpret_cast<const float4*>(p.residual + (int64_t)orow * p.ldc + col);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u)
        *reinterpret_cast<float4*>(cstage + ((rb + u) * EPI_WARPS + ew) * CPAD + lane * 4) = rv[u];
    }
    epi_bar_sync();  // residual chunk complete before the row-per-thread accumulate
  }
  return res_vec;
}

// GEGLU epilogue of a tile of one 128-column chunk packed [64 value | 64 gate] (attention.py:40-43), the accumulator
// staged as CPAD rows.  All accumulator columns this thread needs (16 value + 16 gate of ONE row) are read first; after
// a barrier the staging memory takes the bf16 results (128 B per row), which leave as fully coalesced 16-B-per-lane
// rows: one row per thread straight from registers made every warp store touch 32 different lines.
template <int NCH>
__device__ __forceinline__ void epi_geglu_tile(const EpiParams& p, void* stage, int64_t m0, int n0, int ew, int lg,
                                               int part, int lane) {
  static_assert(NCH == 1, "one 128-column chunk per tile");
  constexpr int W = 64 / EPI_PARTS;
  static_assert(W == 16, "two 16-B units per thread and chunk");
  constexpr int U = NCH * 8;  // 16-B units per staged row
  uint32_t val[NCH][W], gate[NCH][W];
  {
    const uint32_t* arow = reinterpret_cast<const uint32_t*>(stage) + (lg * 32 + lane) * CPAD;
#pragma unroll
    for (int j = 0; j < W; j += 4) {
      const uint4 a = *reinterpret_cast<const uint4*>(arow + part * W + j);
      const uint4 b = *reinterpret_cast<const uint4*>(arow + 64 + part * W + j);
      val[0][j] = a.x; val[0][j + 1] = a.y; val[0][j + 2] = a.z; val[0][j + 3] = a.w;
      gate[0][j] = b.x; gate[0][j + 1] = b.y; gate[0][j + 2] = b.z; gate[0][j + 3] = b.w;
    }
  }
  epi_bar_sync();  // every thread has read its columns: the staging memory takes the bf16 results
  const uint32_t seg_len = (uint32_t)p.seg_len;
  const bool coalesced = (p.ldc % 8 == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0);
  const int r = lg * 32 + lane;  // this thread's row of the tile
  uint4* srow = reinterpret_cast<uint4*>(stage) + r * U;
#pragma unroll
  for (int h = 0; h < NCH; ++h) {
    uint32_t pk[W / 2];
#pragma unroll
    for (int j = 0; j < W; j += 2)
      pk[j / 2] = pack_bf16x2(geglu_fast(__uint_as_float(gate[h][j]), __uint_as_float(val[h][j])),
                              geglu_fast(__uint_as_float(gate[h][j + 1]), __uint_as_float(val[h][j + 1])));
    if (coalesced) {
      // logical unit u of row r lives at (u & ~7) | ((u ^ r) & 7): conflict-free for the row-per-lane stores here
      // and for the unit-per-lane loads below
      const int u0 = h * 8 + part * 2;
      srow[(u0 & ~7) | ((u0 ^ r) & 7)] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
      srow[((u0 + 1) & ~7) | (((u0 + 1) ^ r) & 7)] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
    } else {  // odd leading dimension / unaligned C: 4-byte stores from registers
      const uint32_t m = (uint32_t)m0 + r;
      const int col = (n0 + h * 128) / 2 + part * W;
      if (m < (uint32_t)p.M && col < p.N / 2) {
        int64_t orow = m;
        if (seg_len > 0) { const uint32_t q = m / seg_len; orow = q * (uint32_t)p.seg_stride + (uint32_t)p.seg_off + (m - q * seg_len); }
        __nv_bfloat16* crow = reinterpret_cast<__nv_bfloat16*>(p.C) + orow * p.ldc + col;
#pragma unroll
        for (int j = 0; j < W / 2; ++j) *reinterpret_cast<uint32_t*>(crow + 2 * j) = pk[j];
      }
    }
  }
  if (!coalesced) return;  // uniform over the CTA
  epi_bar_sync();          // tile staged
  constexpr int RPI = 32 / U;                 // rows per warp instruction (4 or 2)
  const int rl = lane / U, u = lane % U;      // this lane's row within the instruction and its 16-B unit
  const bool chunk_ok = (n0 + (u >> 3) * 128) < p.N;
#pragma unroll
  for (int i = 0; i < GM / (EPI_WARPS * RPI); ++i) {
    const int rr = (i * EPI_WARPS + ew) * RPI + rl;
    const uint32_t m = (uint32_t)m0 + rr;
    const uint4 v = reinterpret_cast<const uint4*>(stage)[rr * U + ((u & ~7) | ((u ^ rr) & 7))];
    if (m < (uint32_t)p.M && chunk_ok) {
      int64_t orow = m;
      if (seg_len > 0) { const uint32_t q = m / seg_len; orow = q * (uint32_t)p.seg_stride + (uint32_t)p.seg_off + (m - q * seg_len); }
      *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.C) + orow * p.ldc + n0 / 2 + u * 8) = v;
    }
  }
  epi_bar_sync();          // staging tile free for the next accumulator
}

__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// fp32 chunk (128 rows x 128 columns) through the TMA unit.  Staging = four [128 rows x 128 B] SWIZZLE_128B boxes (one
// per 32-column part): thread (row r, part c) owns exactly one 128-byte swizzled row of box c, so its eight 16-byte
// accesses are conflict-free and need no other thread's data.  Order per chunk:
//   store thread: wait until the previous chunk's bulk stores have READ the boxes; barrier;
//   store thread: bulk-load the residual tile (C itself: x = f(x) + x) into the boxes (mbarrier `bar_res`);
//   all: after the main loop, accumulator quadrants + residual into the boxes (acc_to_stage<true>); barrier;
//        own swizzled row + bias, back into the boxes; fence.proxy.async; barrier;  store thread: four bulk stores.
// part 1, BEFORE the accumulator-ready wait (overlaps the main loop)
__device__ __forceinline__ void epi_tma_begin(const EpiParams& p, uint32_t stage_s, uint32_t bar_res, int m0, int n0,
                                              int ew, int lane) {
  const bool store_thread = ew == 0 && lane == 0;
  if (store_thread) tma_store_wait_read();
  epi_bar_sync();  // the boxes are free (the previous chunk's bulk stores have read them)
  if (p.residual && store_thread) {
    mbar_expect_tx(bar_res, 4 * GM * 128);
#pragma unroll
    for (int c = 0; c < 4; ++c) tma_load_2d(&p.tmC, bar_res, stage_s + c * (GM * 128), n0 + 32 * c, m0);
  }
}
// part 2, after the accumulator (+ residual) has been staged in the boxes
__device__ __forceinline__ void epi_tma_finish(const EpiParams& p, uint8_t* stage, uint32_t stage_s, int m0, int n0,
                                               int ew, int lg, int part, int lane) {
  const int r = lg * 32 + lane;
  float4* box_row = reinterpret_cast<float4*>(stage + part * (GM * 128) + r * 128);
  const int col0 = n0 + part * 32;
  const bool bias_vec = p.bias && (col0 + 31 < p.N) && ((reinterpret_cast<uintptr_t>(p.bias) & 15) == 0);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int pos = j ^ (r & 7);
    float4 o = box_row[pos];
    if (bias_vec) {
      const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias + col0) + j);
      o.x += bv.x; o.y += bv.y; o.z += bv.z; o.w += bv.w;
    } else if (p.bias) {
      const int c = col0 + 4 * j;
      if (c < p.N) o.x += __ldg(p.bias + c);
      if (c + 1 < p.N) o.y += __ldg(p.bias + c + 1);
      if (c + 2 < p.N) o.z += __ldg(p.bias + c + 2);
      if (c + 3 < p.N) o.w += __ldg(p.bias + c + 3);
    }
    box_row[pos] = o;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA unit
  epi_bar_sync();  // whole chunk staged
  if (ew == 0 && lane == 0) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (n0 + 32 * c < p.N) tma_store_2d(&p.tmC, stage_s + c * (GM * 128), n0 + 32 * c, m0);  // OOB rows / columns are clipped
    tma_store_commit();
  }
}

// Writes out one chunk staged as CPAD rows (accumulator + the prefetched residual when res_vec).
template <int EPI>
__device__ __forceinline__ void epi_chunk(const EpiParams& p, float* cstage, int64_t m0, int n0, bool res_vec, int ew,
                                          int lane) {
  const uint32_t seg_len = (uint32_t)p.seg_len;
  // ---- coalesced write-out: one row per warp instruction ----
  constexpr int RPW = GM / EPI_WARPS;  // rows per warp
  const int ncol0 = n0;
  const int nlim = p.N;
  if (EPI == 0) {
    const int col = ncol0 + lane * 4;
    const bool vec = (p.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) && (col + 3 < nlim);
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.bias) {
      if (col < nlim) bv.x = __ldg(p.bias + col);
      if (col + 1 < nlim) bv.y = __ldg(p.bias + col + 1);
      if (col + 2 < nlim) bv.z = __ldg(p.bias + col + 2);
      if (col + 3 < nlim) bv.w = __ldg(p.bias + col + 3);
    }
    // fast path (whole chunk uniform): vector rows, residual already folded in (or absent), full M tile
    const bool fast = (p.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) && (p.N % 4 == 0) &&
                      (res_vec || !p.residual) && (m0 + GM <= p.M) && seg_len == 0;
    if (fast) {
      if (col < nlim) {
        float* cbase = reinterpret_cast<float*>(p.C) + (m0 + ew) * p.ldc + col;
        const float* sbase = cstage + ew * CPAD + lane * 4;
#pragma unroll 1
        for (int rb = 0; rb < RPW; rb += 8) {
          float4 o[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) o[u] = *reinterpret_cast<const float4*>(sbase + (rb + u) * EPI_WARPS * CPAD);
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            o[u].x += bv.x; o[u].y += bv.y; o[u].z += bv.z; o[u].w += bv.w;
            *reinterpret_cast<float4*>(cbase + (int64_t)(rb + u) * EPI_WARPS * p.ldc) = o[u];
          }
        }
      }
    } else
    // general path, 8 rows per batch: all residual loads of a batch are issued before the first store (C may
    // alias the residual -- in-place x = f(x) + x -- so the compiler cannot reorder them itself)
#pragma unroll 1
    for (int rb = 0; rb < RPW; rb += 8) {
      int64_t off[8];
      float4 rv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int r = (rb + u) * EPI_WARPS + ew;
        const uint32_t m = (uint32_t)m0 + r;
        uint32_t orow = m;
        if (seg_len > 0) { const uint32_t q = m / seg_len; orow = q * (uint32_t)p.seg_stride + (uint32_t)p.seg_off + (m - q * seg_len); }
        off[u] = (m < (uint32_t)p.M && col < nlim) ? (int64_t)orow * p.ldc + col : -1;
        rv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!res_vec && vec && p.residual && off[u] >= 0) rv[u] = *reinterpret_cast<const float4*>(p.residual + off[u]);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (off[u] < 0) continue;
        const int r = (rb + u) * EPI_WARPS + ew;
        float4 o = *reinterpret_cast<const float4*>(cstage + r * CPAD + lane * 4);
        o.x += bv.x + rv[u].x; o.y += bv.y + rv[u].y; o.z += bv.z + rv[u].z; o.w += bv.w + rv[u].w;
        float* crow = reinterpret_cast<float*>(p.C) + off[u];
        if (vec) {
          *reinterpret_cast<float4*>(crow) = o;
        } else {  // ragged N / unaligned C: scalar tail
          const float ov[4] = {o.x, o.y, o.z, o.w};
          for (int j = 0; j < 4; ++j)
            if (col + j < nlim) crow[j] = ov[j] + ((p.residual && !res_vec) ? p.residual[off[u] + j] : 0.f);
        }
      }
    }
  } else if (EPI == 3) {
    // bf16 attention operands: lane owns columns [4 lane, 4 lane + 4) of the chunk; a head is 64 columns = 16 lanes, so
    // the squared norm of a (row, head) is a 4-step xor-shuffle over the half warp
    const int col = ncol0 + lane * 4;
    const bool norm = ncol0 < p.norm_cols;   // chunks are 128-aligned and norm_cols % 128 == 0 (checked on the host)
    float4 sc = make_float4(1.f, 1.f, 1.f, 1.f);
    if (norm) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(p.nscale + ((lane * 4) & 63)));
      sc = make_float4(t.x * p.nmul, t.y * p.nmul, t.z * p.nmul, t.w * p.nmul);
    }
#pragma unroll 4
    for (int rr = 0; rr < RPW; ++rr) {
      const int r = rr * EPI_WARPS + ew;
      const uint32_t m = (uint32_t)m0 + r;
      float4 o = *reinterpret_cast<const float4*>(cstage + r * CPAD + lane * 4);
      if (norm) {
        float ss = o.x * o.x + o.y * o.y + o.z * o.z + o.w * o.w;
#pragma unroll
        for (int d = 8; d > 0; d >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, d);
        const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
        o.x = (o.x * inv) * sc.x; o.y = (o.y * inv) * sc.y; o.z = (o.z * inv) * sc.z; o.w = (o.w * inv) * sc.w;
      }
      if (m < (uint32_t)p.M && col < nlim)
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.C) + (int64_t)m * p.ldc + col) =
            make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
    }
  } else {
    // EPI 1: bf16 outputs, 128 columns (4 per lane)
    constexpr int CPL = 4;
    const int col = ncol0 + lane * CPL;
    float bv[CPL];
#pragma unroll
    for (int j = 0; j < CPL; ++j) bv[j] = (p.bias && col + j < nlim) ? __ldg(p.bias + col + j) : 0.f;
    const bool vec = (p.ldc % CPL == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) && (col + CPL - 1 < nlim);
#pragma unroll 4
    for (int rr = 0; rr < RPW; ++rr) {
      const int r = rr * EPI_WARPS + ew;
      const uint32_t m = (uint32_t)m0 + r;
      if (m >= (uint32_t)p.M) break;
      int64_t orow = m;
      if (seg_len > 0) { const uint32_t q = m / seg_len; orow = q * (uint32_t)p.seg_stride + (uint32_t)p.seg_off + (m - q * seg_len); }
      float o[CPL];
#pragma unroll
      for (int j = 0; j < CPL; ++j) o[j] = cstage[r * CPAD + lane * CPL + j] + bv[j];
      __nv_bfloat16* crow = reinterpret_cast<__nv_bfloat16*>(p.C) + orow * p.ldc + col;
      if (vec) {
        *reinterpret_cast<uint2*>(crow) = make_uint2(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]));
      } else {
#pragma unroll
        for (int j = 0; j < CPL; ++j)
          if (col + j < nlim) crow[j] = __float2bfloat16_rn(o[j]);
      }
    }
  }
  epi_bar_sync();  // staging buffer free for the next chunk
}

// ---------------------------------------------------------------------------------------------------
// The kernel: 128 x 128 tiles, four MMA / epilogue warpgroups of one 64 x 64 quadrant each
// ---------------------------------------------------------------------------------------------------
// DUAL: two independent problems (own operands, output, N and K) in ONE launch -- the q and k,v projections of a
// self-attention block, which read different inputs (LayerNorm(x) vs raw x, attention.py:140-144) and are each a
// single wave of tiles: together they make ~3 tiles per CTA, so prologue, epilogue and main loop overlap across tiles
// instead of being paid twice.
template <int EPI, bool DUAL>
__global__ void __launch_bounds__(GTHREADS, 1) gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                const __grid_constant__ CUtensorMap tmB,
                                                                const __grid_constant__ EpiParams p,
                                                                const __grid_constant__ CUtensorMap tmA2,
                                                                const __grid_constant__ CUtensorMap tmB2,
                                                                const __grid_constant__ EpiParams p2) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B atoms need 1024-B alignment
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sA = base, sB = base + GSTAGES * STAGE_BYTES;
  float* cstage = reinterpret_cast<float*>(base_ptr + RING_BYTES);
  const uint32_t bars = base + RING_BYTES + CSTAGE_BYTES;
  // full[s] @ +8s ; empty[s] @ +8(S+s) ; residual landed @ +16S
  const uint32_t bar_res = bars + 16 * GSTAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles1 = p.m_tiles * p.n_tiles;
  const int num_tiles = tiles1 + (DUAL ? p2.m_tiles * p2.n_tiles : 0);
  // tile schedule: round-robin over all tiles (problem 1 first), m-fastest; returns true for a tile of problem 2
  const int my_tiles = (int)blockIdx.x < num_tiles ? (num_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  auto tile_of = [&](int i, int& m0, int& n0) -> bool {
    int tile = (int)blockIdx.x + i * (int)gridDim.x;
    const bool second = DUAL && tile >= tiles1;
    if (second) tile -= tiles1;
    const int mt = second ? p2.m_tiles : p.m_tiles;
    m0 = (tile % mt) * GM;
    n0 = (tile / mt) * GN;
    return second;
  };
  auto kblocks = [&](bool second) { return ((second ? p2.K : p.K) + GK - 1) / GK; };

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    if (DUAL) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA2) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB2) : "memory");
    }
    for (int s = 0; s < GSTAGES; ++s) {
      mbar_init(bars + 8 * s, 1);
      mbar_init(bars + 8 * (GSTAGES + s), EPI_WARPS);  // one arrival per MMA warp
    }
    mbar_init(bar_res, 1);                               // residual tile landed (TMA epilogue)
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();  // everything above (barriers, tensor-map prefetch) overlapped the previous kernel

  if (warp < 4) {
    // ===================== TMA producer =====================
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int it = 0; it < my_tiles; ++it) {
        int m0, n0;
        const bool second = tile_of(it, m0, n0);
        const int num_kb = kblocks(second);
        const CUtensorMap* ma = second ? &tmA2 : &tmA;
        const CUtensorMap* mb = second ? &tmB2 : &tmB;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bars + 8 * (GSTAGES + stage), phase ^ 1);  // slot free (passes immediately on the first lap)
          const uint32_t full = bars + 8 * stage;
          mbar_expect_tx(full, 2 * STAGE_BYTES);
          tma_load_2d(ma, full, sA + stage * STAGE_BYTES, kb * GK, m0);
          tma_load_2d(mb, full, sB + stage * STAGE_BYTES, kb * GK, n0);
          if (++stage == GSTAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue: warps 4..19 =====================
    const int ew = warp - 4;        // 0..15: rows ew, ew+16, ... in the coalesced write-out
    const int lg = warp & 3;        // 32-row group whose rows this warp drains (one row per lane)
    const int part = ew >> 2;       // which quarter of the tile's columns this warp drains
    const int wg = ew >> 2;         // MMA warpgroup: quadrant rows 64 (wg & 1).., columns 64 (wg >> 1)..
    const int rq = (wg & 1) * 64, cq = (wg >> 1) * 64;
    uint32_t res_phase = 0;
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0; it < my_tiles; ++it) {
      int m0, n0;
      const bool second = tile_of(it, m0, n0);
      const EpiParams& pp = second ? p2 : p;
      const bool tma = EPI == 0 && pp.tma_epi;
      bool res_vec = false;
      if (tma) epi_tma_begin(pp, base + RING_BYTES, bar_res, m0, n0, ew, lane);
      else if (EPI == 0) res_vec = epi_residual_prefetch<EPI>(pp, cstage, m0, n0, ew, lane);
      else epi_bar_sync();  // the previous tile's epilogue has left the staging memory
      // ---- main loop: this warpgroup's 64 x 64 quadrant ----
      float d[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) d[i] = 0.f;
      const int num_kb = kblocks(second);
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(bars + 8 * stage, phase);
        const uint64_t da = gmma_desc(sA + stage * STAGE_BYTES + rq * 128);
        const uint64_t db = gmma_desc(sB + stage * STAGE_BYTES + cq * 128);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GK / 16; ++k)  // +32 B per K = 16 inside the 128-B swizzle row => +2 in the address field
          wgmma_m64n64k16_ss<0>(d, da + 2 * k, db + 2 * k, 1u);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bars + 8 * (GSTAGES + stage));  // this warp's reads of the slot are complete
        if (++stage == GSTAGES) { stage = 0; phase ^= 1; }
      }
      // ---- accumulator -> staging (onto the residual where one was staged) ----
      if (tma) {
        if (pp.residual) { mbar_wait(bar_res, res_phase); res_phase ^= 1; }
        acc_to_stage<true>(d, reinterpret_cast<uint8_t*>(cstage), rq, cq, ew & 3, lane, pp.residual != nullptr);
      } else {
        acc_to_stage<false>(d, reinterpret_cast<uint8_t*>(cstage), rq, cq, ew & 3, lane, res_vec);
      }
      epi_bar_sync();  // whole tile staged
      if (tma)
        epi_tma_finish(pp, reinterpret_cast<uint8_t*>(cstage), base + RING_BYTES, m0, n0, ew, lg, part, lane);
      else if (EPI == 2)
        epi_geglu_tile<1>(pp, cstage, m0, n0, ew, lg, part, lane);
      else
        epi_chunk<EPI>(pp, cstage, m0, n0, res_vec, ew, lane);
    }
    if (EPI == 0 && ew == 0 && lane == 0) tma_store_wait_read();  // staging read out before the CTA exits (the writes complete with the grid)
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------
// host side: tensor maps (driver entry point resolved at run time: libphk.so has no link-time libcuda dependency,
// so it also loads on a CPU-only box for the ABI tests)
// ---------------------------------------------------------------------------------------------------

struct MapKey {
  const void* ptr; int64_t rows, cols, ld; int box_rows;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    h = h * 1000003u ^ std::hash<int64_t>()(k.rows);
    h = h * 1000003u ^ std::hash<int64_t>()(k.cols);
    h = h * 1000003u ^ std::hash<int64_t>()(k.ld * 131 + k.box_rows);
    return h;
  }
};

// [rows, cols] bf16, row pitch ld elements; box = [box_rows, 64 cols], SWIZZLE_128B, zero OOB fill
static int get_tensor_map(const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows, CUtensorMap* out) {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  const MapKey key{ptr, rows, cols, ld, box_rows};
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return 0; }
  EncodeTiledFn fn = encode_fn();
  PHK_REQUIRE(fn, PHK_E_UNSUPPORTED, "cuTensorMapEncodeTiled not available from the driver");
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)GK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUtensorMap m;
  const CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PHK_REQUIRE(r == CUDA_SUCCESS, PHK_E_ARG, "cuTensorMapEncodeTiled rejected the operand (alignment / pitch)");
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, m);
  *out = m;
  return 0;
}

// fp32 [rows, cols] output, row pitch ld floats; box = [128 rows, 32 floats = 128 B], SWIZZLE_128B (TMA epilogue)
static int get_c_map(const void* ptr, int64_t rows, int64_t cols, int64_t ld, CUtensorMap* out) {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  const MapKey key{ptr, rows, cols, ld, -32};
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return 0; }
  EncodeTiledFn fn = encode_fn();
  PHK_REQUIRE(fn, PHK_E_UNSUPPORTED, "cuTensorMapEncodeTiled not available from the driver");
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {32, (cuuint32_t)GM};
  const cuuint32_t estr[2] = {1, 1};
  CUtensorMap m;
  const CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PHK_REQUIRE(r == CUDA_SUCCESS, PHK_E_ARG, "cuTensorMapEncodeTiled rejected the output (alignment / pitch)");
  if (cache.size() > 8192) cache.clear();
  cache.emplace(key, m);
  *out = m;
  return 0;
}

// the TMA epilogue applies to plain fp32 outputs: identity row map, 16-byte aligned rows, residual == C (or none)
static int maybe_tma_epilogue(EpiParams& p, int epilogue) {
  p.tma_epi = 0;
  if (epilogue != 0 || p.seg_len != 0 || p.ldc % 4 != 0 || (reinterpret_cast<uintptr_t>(p.C) & 15) != 0 ||
      (p.residual && p.residual != p.C))
    return 0;
  PHK_TRY(get_c_map(p.C, p.M, p.N, p.ldc, &p.tmC));
  p.tma_epi = 1;
  return 0;
}

template <int EPI>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const EpiParams& p, cudaStream_t st) {
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(gemm_bf16_kernel<EPI, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
    mark_configured(&configured_mask);
  }
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = tiles < kNumSMs ? tiles : kNumSMs;
  PHK_CUDA(launch_pdl(gemm_bf16_kernel<EPI, false>, dim3(grid), dim3(GTHREADS), (size_t)(SMEM_TOTAL), st, ta, tb, p, ta, tb, p));
  PHK_LAUNCH_CHECK();
  return 0;
}

template <int EPI>
static int launch_gemm_dual(const CUtensorMap& ta, const CUtensorMap& tb, const EpiParams& p, const CUtensorMap& ta2,
                            const CUtensorMap& tb2, const EpiParams& p2, cudaStream_t st) {
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(gemm_bf16_kernel<EPI, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
    mark_configured(&configured_mask);
  }
  const int tiles = p.m_tiles * p.n_tiles + p2.m_tiles * p2.n_tiles;
  const int grid = tiles < kNumSMs ? tiles : kNumSMs;
  PHK_CUDA(launch_pdl(gemm_bf16_kernel<EPI, true>, dim3(grid), dim3(GTHREADS), (size_t)(SMEM_TOTAL), st, ta, tb, p, ta2, tb2, p2));
  PHK_LAUNCH_CHECK();
  return 0;
}

}  // namespace phk

using namespace phk;

extern "C" int phk_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc, int64_t M,
                             int32_t N, int32_t K, const float* bias, const float* residual, int64_t seg_len,
                             int64_t seg_stride, int64_t seg_off, int32_t epilogue, phk_stream_t s) {
  Prof prof_(FAM_GEMM_BF16, s, 2.0 * (double)M * N * K);
  PHK_REQUIRE(A && W && C, PHK_E_ARG, "phk_gemm_bf16: null pointer");
  PHK_REQUIRE(M >= 0 && N > 0 && K > 0 && lda >= K && ldw >= K, PHK_E_ARG, "phk_gemm_bf16: bad size");
  PHK_REQUIRE(lda % 8 == 0 && ldw % 8 == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(W) & 15) == 0,
              PHK_E_ARG, "phk_gemm_bf16: operands must be 16-byte aligned with leading dimensions multiple of 8 (TMA)");
  PHK_REQUIRE(epilogue >= 0 && epilogue <= 2, PHK_E_ARG, "phk_gemm_bf16: unknown epilogue");
  PHK_REQUIRE(epilogue != 2 || (N % 128 == 0 && !bias && !residual && ldc % 2 == 0 &&
                                (reinterpret_cast<uintptr_t>(C) & 3) == 0),
              PHK_E_ARG, "phk_gemm_bf16: GEGLU epilogue needs N % 128 == 0, an even ldc and no bias/residual");
  PHK_REQUIRE(M < (1LL << 31) - GM, PHK_E_UNSUPPORTED, "phk_gemm_bf16: M too large");
  if (M == 0) return 0;
  CUtensorMap ta, tb;
  PHK_TRY(get_tensor_map(A, M, K, lda, GM, &ta));
  cudaStream_t st = to_stream(s);
  PHK_TRY(get_tensor_map(W, N, K, ldw, GN, &tb));
  EpiParams p{C, ldc, M, N, K, bias, residual, seg_len, seg_stride, seg_off, (int)((M + GM - 1) / GM), (N + GN - 1) / GN};
  PHK_REQUIRE((int64_t)p.m_tiles * p.n_tiles < (1LL << 31), PHK_E_UNSUPPORTED, "phk_gemm_bf16: too many tiles");
  PHK_TRY(maybe_tma_epilogue(p, epilogue));
  if (epilogue == 2) return launch_gemm<2>(ta, tb, p, st);
  if (epilogue == 1) return launch_gemm<1>(ta, tb, p, st);
  return launch_gemm<0>(ta, tb, p, st);
}

// Two independent products C1 = A1 W1^T (+bias1) [M1,N1] and C2 = A2 W2^T (+bias2) [M2,N2] (fp32 outputs) in one
// launch: the q and k,v projections of a self-attention block (attention.py:140-146), or the first-frame and
// rest-frames patch embeddings (cvivit.py:542-549: 16 + 128 tiles, neither of which fills the machine alone).
extern "C" int phk_gemm_bf16_x2(const void* A1, int64_t lda1, const void* W1, int64_t ldw1, float* C1, int64_t ldc1,
                                int64_t M1, int32_t N1, int32_t K1, const float* bias1, const void* A2, int64_t lda2,
                                const void* W2, int64_t ldw2, float* C2, int64_t ldc2, int64_t M2, int32_t N2,
                                int32_t K2, const float* bias2, phk_stream_t s) {
  Prof prof_(FAM_GEMM_BF16, s, 2.0 * ((double)M1 * N1 * K1 + (double)M2 * N2 * K2));
  PHK_REQUIRE(A1 && W1 && C1 && A2 && W2 && C2, PHK_E_ARG, "phk_gemm_bf16_x2: null pointer");
  PHK_REQUIRE(M1 > 0 && M2 > 0 && N1 > 0 && K1 > 0 && N2 > 0 && K2 > 0 && lda1 >= K1 && ldw1 >= K1 && lda2 >= K2 &&
                  ldw2 >= K2, PHK_E_ARG, "phk_gemm_bf16_x2: bad size");
  PHK_REQUIRE(lda1 % 8 == 0 && ldw1 % 8 == 0 && lda2 % 8 == 0 && ldw2 % 8 == 0 &&
                  ((reinterpret_cast<uintptr_t>(A1) | reinterpret_cast<uintptr_t>(W1) | reinterpret_cast<uintptr_t>(A2) |
                    reinterpret_cast<uintptr_t>(W2)) & 15) == 0,
              PHK_E_ARG, "phk_gemm_bf16_x2: operands must be 16-byte aligned with leading dimensions multiple of 8 (TMA)");
  PHK_REQUIRE(M1 < (1LL << 31) - 2 * GM && M2 < (1LL << 31) - 2 * GM, PHK_E_UNSUPPORTED, "phk_gemm_bf16_x2: M too large");
  CUtensorMap ta, tb, ta2, tb2;
  PHK_TRY(get_tensor_map(A1, M1, K1, lda1, GM, &ta));
  PHK_TRY(get_tensor_map(A2, M2, K2, lda2, GM, &ta2));
  PHK_TRY(get_tensor_map(W1, N1, K1, ldw1, GN, &tb));
  PHK_TRY(get_tensor_map(W2, N2, K2, ldw2, GN, &tb2));
  EpiParams p{C1, ldc1, M1, N1, K1, bias1, nullptr, 0, 0, 0, (int)((M1 + GM - 1) / GM), (N1 + GN - 1) / GN};
  EpiParams p2{C2, ldc2, M2, N2, K2, bias2, nullptr, 0, 0, 0, (int)((M2 + GM - 1) / GM), (N2 + GN - 1) / GN};
  PHK_REQUIRE((int64_t)p.m_tiles * p.n_tiles + (int64_t)p2.m_tiles * p2.n_tiles < (1LL << 31), PHK_E_UNSUPPORTED,
              "phk_gemm_bf16_x2: too many tiles");
  // (measured: the bulk-store epilogue does not pay for the two-problem launch -- 16.2 vs 15.5 us -- so it stays off)
  return launch_gemm_dual<0>(ta, tb, p, ta2, tb2, p2, to_stream(s));
}

// The q and k,v projections of a self-attention block (attention.py:140-157) in one launch, written as the bf16 operands
// of the attention core: Qn[M, I] = normalize_per_head(xn Wq^T) * q_scale * sim_scale, KVn[M, 2I] = [normalize_per_head(
// xraw Wk^T) * k_scale | xraw Wv^T].  dim_head 64, I % 128 == 0.  Replaces fp32 q / kv round trips + a separate
// normalisation pass.
extern "C" int phk_gemm_bf16_qkv(const void* xn, const void* xraw, int64_t lda, const void* Wq, const void* Wkv, int64_t ldw,
                                 void* Qn, void* KVn, int64_t M, int32_t I, int32_t K, const float* q_scale,
                                 const float* k_scale, float sim_scale, phk_stream_t s) {
  Prof prof_(FAM_GEMM_BF16, s, 2.0 * (double)M * 3.0 * I * K);
  PHK_REQUIRE(xn && xraw && Wq && Wkv && Qn && KVn && q_scale && k_scale, PHK_E_ARG, "phk_gemm_bf16_qkv: null pointer");
  PHK_REQUIRE(M > 0 && I > 0 && I % 128 == 0 && K > 0 && lda >= K && ldw >= K, PHK_E_ARG,
              "phk_gemm_bf16_qkv: heads * 64 must be a multiple of 128");
  PHK_REQUIRE(lda % 8 == 0 && ldw % 8 == 0 &&
                  ((reinterpret_cast<uintptr_t>(xn) | reinterpret_cast<uintptr_t>(xraw) | reinterpret_cast<uintptr_t>(Wq) |
                    reinterpret_cast<uintptr_t>(Wkv) | reinterpret_cast<uintptr_t>(q_scale) |
                    reinterpret_cast<uintptr_t>(k_scale)) & 15) == 0 &&
                  ((reinterpret_cast<uintptr_t>(Qn) | reinterpret_cast<uintptr_t>(KVn)) & 7) == 0,
              PHK_E_ARG, "phk_gemm_bf16_qkv: operands must be 16-byte aligned with leading dimensions multiple of 8 (TMA)");
  PHK_REQUIRE(M < (1LL << 31) - 2 * GM, PHK_E_UNSUPPORTED, "phk_gemm_bf16_qkv: M too large");
  CUtensorMap ta, tb, ta2, tb2;
  PHK_TRY(get_tensor_map(xn, M, K, lda, GM, &ta));
  PHK_TRY(get_tensor_map(xraw, M, K, lda, GM, &ta2));
  PHK_TRY(get_tensor_map(Wq, I, K, ldw, GN, &tb));
  PHK_TRY(get_tensor_map(Wkv, 2 * I, K, ldw, GN, &tb2));
  EpiParams p{Qn, I, M, I, K, nullptr, nullptr, 0, 0, 0, (int)((M + GM - 1) / GM), I / GN};
  EpiParams p2{KVn, 2 * (int64_t)I, M, 2 * I, K, nullptr, nullptr, 0, 0, 0, (int)((M + GM - 1) / GM), 2 * I / GN};
  p.tma_epi = 0; p.nscale = q_scale; p.norm_cols = I; p.nmul = sim_scale;
  p2.tma_epi = 0; p2.nscale = k_scale; p2.norm_cols = I; p2.nmul = 1.0f;
  PHK_REQUIRE((int64_t)p.m_tiles * p.n_tiles + (int64_t)p2.m_tiles * p2.n_tiles < (1LL << 31), PHK_E_UNSUPPORTED,
              "phk_gemm_bf16_qkv: too many tiles");
  return launch_gemm_dual<3>(ta, tb, p, ta2, tb2, p2, to_stream(s));
}

// The q projection of a cross-attention block (attention.py:139, 153-157) written as the bf16 operand of the attention
// core: Qn[M, I] = normalize_per_head(xn Wq^T) * q_scale * sim_scale (epilogue 3 on one problem).  dim_head 64, I % 128 == 0.
extern "C" int phk_gemm_bf16_qnorm(const void* xn, int64_t lda, const void* Wq, int64_t ldw, void* Qn, int64_t M, int32_t I,
                                   int32_t K, const float* q_scale, float sim_scale, phk_stream_t s) {
  Prof prof_(FAM_GEMM_BF16, s, 2.0 * (double)M * I * K);
  PHK_REQUIRE(xn && Wq && Qn && q_scale, PHK_E_ARG, "phk_gemm_bf16_qnorm: null pointer");
  PHK_REQUIRE(M > 0 && I > 0 && I % 128 == 0 && K > 0 && lda >= K && ldw >= K, PHK_E_ARG,
              "phk_gemm_bf16_qnorm: heads * 64 must be a multiple of 128");
  PHK_REQUIRE(lda % 8 == 0 && ldw % 8 == 0 &&
                  ((reinterpret_cast<uintptr_t>(xn) | reinterpret_cast<uintptr_t>(Wq) | reinterpret_cast<uintptr_t>(q_scale)) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(Qn) & 7) == 0,
              PHK_E_ARG, "phk_gemm_bf16_qnorm: operands must be 16-byte aligned with leading dimensions multiple of 8 (TMA)");
  PHK_REQUIRE(M < (1LL << 31) - 2 * GM, PHK_E_UNSUPPORTED, "phk_gemm_bf16_qnorm: M too large");
  CUtensorMap ta, tb;
  PHK_TRY(get_tensor_map(xn, M, K, lda, GM, &ta));
  PHK_TRY(get_tensor_map(Wq, I, K, ldw, GN, &tb));
  EpiParams p{Qn, I, M, I, K, nullptr, nullptr, 0, 0, 0, (int)((M + GM - 1) / GM), I / GN};
  p.tma_epi = 0; p.nscale = q_scale; p.norm_cols = I; p.nmul = sim_scale;
  return launch_gemm<3>(ta, tb, p, to_stream(s));
}
