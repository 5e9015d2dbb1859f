// bf16 GEMM on the Hopper tensor cores (sm_90a, wgmma):
//   C[map(m), n] = sum_k A[m,k] * W[n,k]  (+bias) (+residual)        nn.Linear semantics
// A, W bf16, K-major (row-major [rows, K]); fp32 accumulation in registers.
//
// gemm_bf16_kernel<EPI, DUAL> behind phk_gemm_bf16 / phk_gemm_bf16_x2 / _qkv / _qnorm, DUAL = two independent problems
// in one launch.  Persistent (one CTA per SM, 128 x 128 tiles or 64 x 128 units, static round-robin scheduler,
// m-fastest so concurrent CTAs share the W tile in L2 while the A panel stays L2-resident).  Two bodies:
// * quadrant (bf16 single-problem instances <1, false> and <3, false>, 640 threads):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor.2d (SWIZZLE_128B) stages 128x64 A and W tiles into
//                   a 4-deep shared-memory ring; out-of-bounds rows / the K tail are zero-filled by the TMA unit.
//   warpgroups 1..4 each multiplies one 64 x 64 quadrant of the tile (wgmma.m64n64k16, both operands from shared
//                   memory), writes it into the epilogue's staging layout, and then all sixteen warps run the epilogue
//                   (four per 32-row group, each a quarter of the columns) while the producer fills the ring for the
//                   next tile.
// * ping-pong (384 threads; see gemm_pingpong below): two MMA warpgroups take whole units in turn as m64n128k16 row
//   halves and run the epilogue while the other one runs its main loop.  128 x 128 tiles for the two-problem instances
//   and gemm_bf16_geglu_kernel; 64 x 128 units for the fp32 single-problem instance <0, false> (out-projection, FF2).
// Epilogues: 0 fp32 (+residual, +bias, row map), (acc + residual) + bias -- single problem: through the TMA unit when
//              the row map is the identity: the residual tile is bulk-loaded into the warpgroup's SWIZZLE_128B staging
//              boxes during the main loop and the result bulk-stored from them; otherwise from the registers.  Two
//              problems: fp32 (+bias) from the registers.
//            1 bf16 (+bias)
//            2 GEGLU (attention.py:40-43) on W rows packed [64 value rows | 64 gate rows] per 128-column tile ->
//              bf16 [M, N/2], fitted sigmoid-form GELU: gemm_bf16_geglu_kernel (ping-pong)
//            3 q / k,v attention operands (per-head l2 normalisation, bf16): staged (one problem) or from the registers
//              (two problems), rounded alike.
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
  int m_tiles, n_tiles;  // row and column units of the launch (64 or 128 rows, 128 columns)
  // fp32 epilogue through the TMA unit (identity row map, C 16-B aligned, residual == C or none): C as a tensor map
  // with [64 rows x 32 floats] SWIZZLE_128B boxes; the residual tile is bulk-LOADED into the staging boxes while the
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
// epilogue's staging rows of CPAD floats.
__device__ __forceinline__ void acc_to_stage(const float (&d)[32], float* stage, int rq, int cq, int w, int lane) {
  const int r0 = rq + 16 * w + (lane >> 2);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = cq + 8 * j + 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(stage + (r0 + 8 * h) * CPAD + c) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
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

// Per-head l2 normalisation of epilogue 3, shared by the staged and the register epilogue so that both round alike: the
// squared norm of four consecutive columns c0..c3 of a head is fma(c3, c3, fma(c2, c2, fma(c0, c0, c1 * c1))), the
// head's 16 such partials are summed as an xor-butterfly over 8, 4, 2, 1, and each column becomes (c * inv) * scale.
__device__ __forceinline__ float head_sumsq_first(float c0, float c1) { return __fmaf_rn(c0, c0, __fmul_rn(c1, c1)); }
__device__ __forceinline__ float head_sumsq_next(float c2, float c3, float s) {
  return __fmaf_rn(c3, c3, __fmaf_rn(c2, c2, s));
}
__device__ __forceinline__ float head_inv_norm(float ss) { return 1.0f / fmaxf(sqrtf(ss), 1e-12f); }
__device__ __forceinline__ float head_scale(float c, float inv, float sc) { return __fmul_rn(__fmul_rn(c, inv), sc); }

// ---------------------------------------------------------------------------------------------------
// Epilogue pieces.  A "chunk" is the tile's 128 rows x 128 accumulator columns, staged in shared memory by
// acc_to_stage.
// ---------------------------------------------------------------------------------------------------

__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// Writes out one chunk staged as CPAD rows (quadrant body: bf16 epilogues 1 and 3).
template <int EPI>
__device__ __forceinline__ void epi_chunk(const EpiParams& p, float* cstage, int64_t m0, int n0, int ew, int lane) {
  static_assert(EPI == 1 || EPI == 3, "the fp32 epilogue runs on the ping-pong body");
  const uint32_t seg_len = (uint32_t)p.seg_len;
  // ---- coalesced write-out: one row per warp instruction ----
  constexpr int RPW = GM / EPI_WARPS;  // rows per warp
  const int ncol0 = n0;
  const int nlim = p.N;
  if (EPI == 3) {
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
        float ss = head_sumsq_next(o.z, o.w, head_sumsq_first(o.x, o.y));
#pragma unroll
        for (int d = 8; d > 0; d >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, d);
        const float inv = head_inv_norm(ss);
        o.x = head_scale(o.x, inv, sc.x); o.y = head_scale(o.y, inv, sc.y);
        o.z = head_scale(o.z, inv, sc.z); o.w = head_scale(o.w, inv, sc.w);
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
// Quadrant body (bf16 single-problem instances): 128 x 128 tiles, four MMA / epilogue warpgroups of one 64 x 64 quadrant
// each
// ---------------------------------------------------------------------------------------------------
template <int EPI>
__device__ __forceinline__ void gemm_quadrant(const CUtensorMap& tmA, const CUtensorMap& tmB, const EpiParams& p) {
  static_assert(EPI == 1 || EPI == 3, "the fp32 epilogue runs on the ping-pong body");
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B atoms need 1024-B alignment
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sA = base, sB = base + GSTAGES * STAGE_BYTES;
  float* cstage = reinterpret_cast<float*>(base_ptr + RING_BYTES);
  const uint32_t bars = base + RING_BYTES + CSTAGE_BYTES;  // full[s] @ +8s ; empty[s] @ +8(S+s)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = p.m_tiles * p.n_tiles;
  // tile schedule: round-robin, m-fastest
  const int my_tiles = (int)blockIdx.x < num_tiles ? (num_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  auto tile_of = [&](int i, int& m0, int& n0) {
    const int tile = (int)blockIdx.x + i * (int)gridDim.x;
    m0 = (tile % p.m_tiles) * GM;
    n0 = (tile / p.m_tiles) * GN;
  };
  const int num_kb = (p.K + GK - 1) / GK;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < GSTAGES; ++s) {
      mbar_init(bars + 8 * s, 1);
      mbar_init(bars + 8 * (GSTAGES + s), EPI_WARPS);  // one arrival per MMA warp
    }
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
        tile_of(it, m0, n0);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bars + 8 * (GSTAGES + stage), phase ^ 1);  // slot free (passes immediately on the first lap)
          const uint32_t full = bars + 8 * stage;
          mbar_expect_tx(full, 2 * STAGE_BYTES);
          tma_load_2d(&tmA, full, sA + stage * STAGE_BYTES, kb * GK, m0);
          tma_load_2d(&tmB, full, sB + stage * STAGE_BYTES, kb * GK, n0);
          if (++stage == GSTAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue: warps 4..19 =====================
    const int ew = warp - 4;        // 0..15: rows ew, ew+16, ... in the coalesced write-out
    const int wg = ew >> 2;         // MMA warpgroup: quadrant rows 64 (wg & 1).., columns 64 (wg >> 1)..
    const int rq = (wg & 1) * 64, cq = (wg >> 1) * 64;
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0; it < my_tiles; ++it) {
      int m0, n0;
      tile_of(it, m0, n0);
      epi_bar_sync();  // the previous tile's epilogue has left the staging memory
      // ---- main loop: this warpgroup's 64 x 64 quadrant ----
      float d[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) d[i] = 0.f;
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
      acc_to_stage(d, cstage, rq, cq, ew & 3, lane);
      epi_bar_sync();  // whole tile staged
      epi_chunk<EPI>(p, cstage, m0, n0, ew, lane);
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------
// Ping-pong body: the GEGLU products (FF1 of every feed-forward block, 22 column tiles), the two-problem launches
// (q + k,v projections, patch embeddings) and the fp32 single-problem products (out-projection and FF2 + residual)
// ---------------------------------------------------------------------------------------------------
// Warpgroup 0 is the TMA producer (one thread; the warpgroup gives its registers away to the MMA warpgroups) feeding a
// GG_STAGES-deep ring in the order the CTA's units are consumed.  Warpgroups 1 and 2 take the CTA's units in turn: each
// multiplies a whole UM x 128 unit as UM / 64 m64n128k16 row halves that share every W slice (6 KB of operands per 64
// tensor-core clocks instead of 4 KB per 32 for a 64 x 64 quadrant), keeps one k-block of MMAs in flight, and runs the
// epilogue while the other warpgroup runs the next unit's main loop, so only the CTA's last epilogue is exposed.  A
// named-barrier handshake orders the main loops, so the two warpgroups never interleave their MMAs.  Per output element
// the k-order (k-blocks of 64 in order, k = 16 steps in order) is that of the quadrant body.
// UM = 128 for the GEGLU and two-problem products.  UM = 64 for the fp32 single-problem products: at 4608 x 512 the
// 288 units make 2.2 per CTA (a makespan of 1.5 tile-times) where 144 128-row tiles make 1.1 (two tile-times, the
// machine 55 % busy).  The price: 24 KB of operands per k-block for half a tile's MMAs (32 KB for a whole 128-row
// tile), which costs at long K (the single patch embedding, K = 6144, is slower than on 128-row tiles).
// DUAL: two independent problems (own operands, output, N and K) in ONE launch, tiles of problem 1 first.  The q and
// k,v projections of a self-attention block read different inputs (LayerNorm(x) vs raw x, attention.py:140-144) and
// are each a single wave of tiles; together they make 3-4 tiles per CTA.
constexpr int GG_STAGES = 6;
constexpr int GG_THREADS = 384;
constexpr int GG_PRODUCER_REGS = 40, GG_CONSUMER_REGS = 232;  // 128 x 40 + 256 x 232 <= 64 K registers
constexpr int UNIT_M = 64;      // rows of a unit of the fp32 single-problem products
constexpr int GG_BAR_TURN = 1;  // named barriers 1, 2: main-loop turn of MMA warpgroup 0, 1
constexpr int GG_BAR_EPI = 3;   // named barriers 3, 4: staging area of MMA warpgroup 0, 1
// Shared memory of a ping-pong launch: the ring, then one staging area per MMA warpgroup, then the barriers
template <int UM, class Epilogue>
constexpr int pingpong_smem() {
  return GG_STAGES * (UM * GK * 2 + STAGE_BYTES) + 2 * Epilogue::kStageBytes + 128 /*barriers*/ +
         1024 /*manual 1024-B alignment*/;
}

// The accumulator of a ping-pong unit: acc[h][4j + 2i + e] = (row 64h + 16w + lane/4 + 8i, column 8j + 2(lane%4) + e).
template <int UM>
using PingPongAcc = float[UM / 64][64];

// An MMA warp as its epilogue sees it: warp w of MMA warpgroup wg, and the warpgroup's staging area in shared memory
// (Epilogue::kStageBytes at `stage`, shared address stage_s) with the mbarrier `bar` of its bulk loads (phase `phase`).
struct PingPongWarp {
  int wg, w, lane;
  uint8_t* stage;
  uint32_t stage_s, bar, phase;
};

// Epilogues straight from the accumulator registers: no staging area, nothing to load ahead of the main loop.
struct RegisterEpilogue {
  static constexpr int kStageBytes = 0;
  __device__ __forceinline__ void prefetch(const EpiParams&, int, int, const PingPongWarp&) const {}
};
constexpr int GG_SMEM_TOTAL = pingpong_smem<128, RegisterEpilogue>();

template <bool DUAL, int UM, class Epilogue>
__device__ __forceinline__ void gemm_pingpong(const CUtensorMap& tmA, const CUtensorMap& tmB, const EpiParams& p,
                                              const CUtensorMap& tmA2, const CUtensorMap& tmB2, const EpiParams& p2,
                                              const Epilogue& epilogue) {
  constexpr int A_BYTES = UM * GK * 2;  // the A box of a unit; the W box is STAGE_BYTES
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;  // SWIZZLE_128B atoms need 1024-B alignment
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sA = base, sB = base + GG_STAGES * A_BYTES;
  const uint32_t sC = sB + GG_STAGES * STAGE_BYTES;                // staging areas (1024-B aligned)
  // full[s] @ +8s ; empty[s] @ +8(S+s) ; staging-area load of MMA warpgroup g landed @ +16S + 8g
  const uint32_t bars = sC + 2 * Epilogue::kStageBytes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles1 = p.m_tiles * p.n_tiles;
  const int num_tiles = tiles1 + (DUAL ? p2.m_tiles * p2.n_tiles : 0);
  const int my_tiles = (int)blockIdx.x < num_tiles ? (num_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  // round-robin over all tiles (problem 1 first), m-fastest; returns true for a tile of problem 2
  auto tile_of = [&](int i, int& m0, int& n0) -> bool {
    int tile = (int)blockIdx.x + i * (int)gridDim.x;
    const bool second = DUAL && tile >= tiles1;
    if (second) tile -= tiles1;
    const int mt = second ? p2.m_tiles : p.m_tiles;
    m0 = (tile % mt) * UM;
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
    for (int s = 0; s < GG_STAGES; ++s) {
      mbar_init(bars + 8 * s, 1);
      mbar_init(bars + 8 * (GG_STAGES + s), 4);  // one arrival per warp of the consuming MMA warpgroup
    }
    if (Epilogue::kStageBytes > 0) {
      mbar_init(bars + 16 * GG_STAGES, 1);
      mbar_init(bars + 16 * GG_STAGES + 8, 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();  // everything above (barriers, tensor-map prefetch) overlapped the previous kernel

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<GG_PRODUCER_REGS>();
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
          mbar_wait(bars + 8 * (GG_STAGES + stage), phase ^ 1);  // slot free (passes immediately on the first lap)
          const uint32_t full = bars + 8 * stage;
          mbar_expect_tx(full, A_BYTES + STAGE_BYTES);
          tma_load_2d(ma, full, sA + stage * A_BYTES, kb * GK, m0);
          tma_load_2d(mb, full, sB + stage * STAGE_BYTES, kb * GK, n0);
          if (++stage == GG_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue: warpgroup wg takes the CTA's units wg, wg + 2, ... =====================
    setmaxnreg_inc<GG_CONSUMER_REGS>();
    const int wg = (warp >> 2) - 1;
    const int w = warp & 3;
    PingPongWarp pw{wg, w, lane, base_ptr + (sC - base) + wg * Epilogue::kStageBytes, sC + wg * Epilogue::kStageBytes,
                    bars + 16 * GG_STAGES + 8 * wg, 0};
    int stage = 0;
    uint32_t phase = 0;
    for (int it = 0; it < my_tiles; ++it) {
      int m0, n0;
      const bool second = tile_of(it, m0, n0);
      const int num_kb = kblocks(second);
      if ((it & 1) != wg) {  // the other warpgroup's unit: skip its k-blocks in the ring
        stage += num_kb;
        while (stage >= GG_STAGES) { stage -= GG_STAGES; phase ^= 1; }
        continue;
      }
      epilogue.prefetch(second ? p2 : p, m0, n0, pw);  // e.g. the residual tile, while this warpgroup waits and runs
      if (it > 0) named_bar_sync(GG_BAR_TURN + wg, 256);  // the other warpgroup has issued unit it - 1
      PingPongAcc<UM> acc;
      int prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(bars + 8 * stage, phase);
        const uint64_t da = gmma_desc(sA + stage * A_BYTES);
        const uint64_t db = gmma_desc(sB + stage * STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GK / 16; ++k) {  // +32 B per K = 16 inside the 128-B swizzle row => +2 in the address field
          const uint32_t accumulate = (kb > 0 || k > 0) ? 1u : 0u;
#pragma unroll
          for (int h = 0; h < UM / 64; ++h)  // row half h: +64 rows = +8 KB = +512 in the address field
            wgmma_m64n128k16_ss(acc[h], da + 512 * h + 2 * k, db + 2 * k, accumulate);
        }
        wgmma_commit();
        wgmma_wait<1>();  // k-block kb - 1 retired: its slot can be refilled while kb runs
        if (kb > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(bars + 8 * (GG_STAGES + prev));
        }
        prev = stage;
        if (++stage == GG_STAGES) { stage = 0; phase ^= 1; }
      }
      if (it + 1 < my_tiles) named_bar_arrive(GG_BAR_TURN + (wg ^ 1), 256);  // the other warpgroup's turn
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(bars + 8 * (GG_STAGES + prev));
      epilogue(second ? p2 : p, acc, m0, n0, pw);
    }
    // the last unit's bulk stores have read the staging area before the CTA exits (the writes complete with the grid)
    if (Epilogue::kStageBytes > 0 && w == 0 && lane == 0) tma_store_wait_read();
  }
  __syncthreads();
}

// GEGLU of the [64 value | 64 gate] tile -> bf16 columns n0/2 + 8j + 2(lane%4) + e, j < 8: value column c and gate
// column c + 64 of a row are held by the same lane (N % 128 == 0, even ldc and 4-byte aligned C: checked on the host)
struct GegluEpilogue : RegisterEpilogue {
  __device__ __forceinline__ void operator()(const EpiParams& p, const PingPongAcc<128>& acc, int m0, int n0,
                                             const PingPongWarp& pw) const {
    const int w = pw.w, lane = pw.lane;
    __nv_bfloat16* C = reinterpret_cast<__nv_bfloat16*>(p.C);
    const int oc = n0 / 2 + 2 * (lane & 3);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const uint32_t m = (uint32_t)m0 + 64 * (r >> 1) + 16 * w + (lane >> 2) + 8 * (r & 1);
      if (m >= (uint32_t)p.M) continue;
      int64_t orow = m;
      const uint32_t seg_len = (uint32_t)p.seg_len;
      if (seg_len > 0) { const uint32_t q = m / seg_len; orow = q * (uint32_t)p.seg_stride + (uint32_t)p.seg_off + (m - q * seg_len); }
      const float* a = acc[r >> 1] + 2 * (r & 1);
      uint32_t* crow = reinterpret_cast<uint32_t*>(C + orow * p.ldc + oc);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        crow[4 * j] = pack_bf16x2(geglu_fast(a[4 * (j + 8)], a[4 * j]), geglu_fast(a[4 * (j + 8) + 1], a[4 * j + 1]));
    }
  }
};

// Epilogue 3 from the accumulator: bit-identical to epi_chunk<3>.  There lane L of a half-warp owns head-local columns
// 4L..4L+3; here lane quad position t holds columns 8jj + 2t + {0, 1} of a head (jj < 8), so the four columns of L sit
// in quad lanes t = 2(L & 1) (first two) and t + 1 (last two) at jj = L >> 1.  The first lane's partial goes to the
// second, which adds its two squares: the odd quad lanes then hold the staged path's 4-column partials.  Its xor-butterfly
// over L ^ 8, L ^ 4, L ^ 2 pairs registers jj ^ 4, jj ^ 2, jj ^ 1 of one lane, and L ^ 1 pairs quad lanes 1 and 3; float
// addition is commutative, so every level rounds as there.  Columns >= norm_cols (the value half of k,v) are only
// converted.  bf16 output, no bias, identity row map, N % 128 == 0 and 8-byte aligned C (checked on the host).
struct QkNormEpilogue : RegisterEpilogue {
  __device__ __forceinline__ void operator()(const EpiParams& p, const PingPongAcc<128>& acc, int m0, int n0,
                                             const PingPongWarp& pw) const {
    const int w = pw.w, lane = pw.lane;
    const int t = lane & 3;
    const bool norm = n0 < p.norm_cols;  // tiles are 128-aligned and norm_cols % 128 == 0
    float2 sc[8];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) sc[jj] = make_float2(1.f, 1.f);
    if (norm) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const float2 s = __ldg(reinterpret_cast<const float2*>(p.nscale + 8 * jj + 2 * t));
        sc[jj] = make_float2(s.x * p.nmul, s.y * p.nmul);
      }
    }
    __nv_bfloat16* C = reinterpret_cast<__nv_bfloat16*>(p.C);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const uint32_t m = (uint32_t)m0 + 64 * (r >> 1) + 16 * w + (lane >> 2) + 8 * (r & 1);
      const float* a = acc[r >> 1] + 2 * (r & 1);
      uint32_t* crow = reinterpret_cast<uint32_t*>(C + (int64_t)m * p.ldc + n0 + 2 * t);
#pragma unroll
      for (int hd = 0; hd < 2; ++hd) {
        float inv = 1.f;
        if (norm) {  // tile-uniform: every lane of the warp takes part in the shuffles, whatever its row
          float s[8];
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const float c0 = a[4 * (8 * hd + jj)], c1 = a[4 * (8 * hd + jj) + 1];
            const float first = __shfl_xor_sync(0xffffffffu, head_sumsq_first(c0, c1), 1);
            s[jj] = head_sumsq_next(c0, c1, first);
          }
          float ss = ((s[0] + s[4]) + (s[2] + s[6])) + ((s[1] + s[5]) + (s[3] + s[7]));
          ss += __shfl_xor_sync(0xffffffffu, ss, 2);
          ss = __shfl_sync(0xffffffffu, ss, lane | 1);
          inv = head_inv_norm(ss);
        }
        if (m < (uint32_t)p.M) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            float x = a[4 * (8 * hd + jj)], y = a[4 * (8 * hd + jj) + 1];
            if (norm) { x = head_scale(x, inv, sc[jj].x); y = head_scale(y, inv, sc[jj].y); }
            crow[4 * (8 * hd + jj)] = pack_bf16x2(x, y);
          }
        }
      }
    }
  }
};

// Epilogue 0 from the accumulator: fp32 (acc + residual) + bias with the row map; float2 accesses, scalar ones for
// ragged N or a C / residual that is not 8-byte aligned.  SINGLE: the single-problem launches that the TMA unit cannot
// serve (Fp32StagedEpilogue), with residual and row map; otherwise the two-problem launch, which has neither.  C may
// alias the residual (in-place x = f(x) + x): every element is read and written by the same thread.
template <bool SINGLE>
struct Fp32Epilogue : RegisterEpilogue {
  template <int H>  // row halves of the unit
  __device__ __forceinline__ void operator()(const EpiParams& p, const float (&acc)[H][64], int m0, int n0,
                                             const PingPongWarp& pw) const {
    const int c0 = n0 + 2 * (pw.lane & 3);
    float2 bv[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = c0 + 8 * j;
      bv[j].x = (p.bias && c < p.N) ? __ldg(p.bias + c) : 0.f;
      bv[j].y = (p.bias && c + 1 < p.N) ? __ldg(p.bias + c + 1) : 0.f;
    }
    const float* res = SINGLE ? p.residual : nullptr;
    const bool vec = (p.ldc % 2 == 0) && (((reinterpret_cast<uintptr_t>(p.C) | reinterpret_cast<uintptr_t>(res)) & 7) == 0);
    const uint32_t seg_len = SINGLE ? (uint32_t)p.seg_len : 0u;
#pragma unroll
    for (int r = 0; r < 2 * H; ++r) {
      const uint32_t m = (uint32_t)m0 + 64 * (r >> 1) + 16 * pw.w + (pw.lane >> 2) + 8 * (r & 1);
      if (m >= (uint32_t)p.M) continue;
      uint32_t orow = m;
      if (seg_len > 0) { const uint32_t q = m / seg_len; orow = q * (uint32_t)p.seg_stride + (uint32_t)p.seg_off + (m - q * seg_len); }
      const float* a = acc[r >> 1] + 2 * (r & 1);
      const int64_t off = (int64_t)orow * p.ldc + c0;
      float* crow = reinterpret_cast<float*>(p.C) + off;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float2 o = make_float2(a[4 * j], a[4 * j + 1]);
        const int c = c0 + 8 * j;
        if (vec && c + 1 < p.N) {
          if (res) { const float2 rv = *reinterpret_cast<const float2*>(res + off + 8 * j); o.x += rv.x; o.y += rv.y; }
          o.x += bv[j].x; o.y += bv[j].y;
          *reinterpret_cast<float2*>(crow + 8 * j) = o;
        } else {
          if (c < p.N) crow[8 * j] = (res ? o.x + res[off + 8 * j] : o.x) + bv[j].x;
          if (c + 1 < p.N) crow[8 * j + 1] = (res ? o.y + res[off + 8 * j + 1] : o.y) + bv[j].y;
        }
      }
    }
  }
};

// Epilogue 0 of the single-problem launch (64-row units): fp32 (acc + residual) + bias through the TMA unit when the
// row map is the identity, C is 16-byte aligned with ldc % 4 == 0 and the residual is C or absent (p.tma_epi); every
// other call takes Fp32Epilogue.  The staging area of an MMA warpgroup is four [64 rows x 32 floats = 128 B]
// SWIZZLE_128B boxes, the unit's 64 x 128 fp32 output.  Per unit:
//   prefetch (before the warpgroup's turn): the store thread waits until its previous unit's bulk stores have read the
//     area and bulk-loads the residual tile (C itself) into it -- the load runs under this unit's main loop;
//   epilogue: wait for the residual (or, without one, for the store thread's all-clear); each thread adds its
//     accumulator fragment onto the residual in the boxes, then the bias; fence.proxy.async; warpgroup barrier; the
//     store thread bulk-stores the boxes (the TMA unit clips rows >= M and columns >= N) and moves on.
struct Fp32StagedEpilogue {
  static constexpr int kStageBytes = 64 * 128 * 4;
  static constexpr int kBoxBytes = 64 * 128;
  __device__ __forceinline__ void prefetch(const EpiParams& p, int m0, int n0, const PingPongWarp& pw) const {
    if (!p.tma_epi || pw.w != 0 || pw.lane != 0) return;
    tma_store_wait_read();
    if (p.residual) {
      mbar_expect_tx(pw.bar, kStageBytes);
#pragma unroll
      for (int c = 0; c < 4; ++c) tma_load_2d(&p.tmC, pw.bar, pw.stage_s + c * kBoxBytes, n0 + 32 * c, m0);
    }
  }
  __device__ __forceinline__ void operator()(const EpiParams& p, const PingPongAcc<64>& acc, int m0, int n0,
                                             PingPongWarp& pw) const {
    if (!p.tma_epi) { Fp32Epilogue<true>{}(p, acc, m0, n0, pw); return; }
    const int t = pw.lane & 3;
    float2 bv[16];
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = n0 + 8 * j + 2 * t;
        bv[j].x = c < p.N ? __ldg(p.bias + c) : 0.f;
        bv[j].y = c + 1 < p.N ? __ldg(p.bias + c + 1) : 0.f;
      }
    }
    if (p.residual) {
      mbar_wait(pw.bar, pw.phase);
      pw.phase ^= 1;
    } else {
      named_bar_sync(GG_BAR_EPI + pw.wg, 128);  // the store thread has seen the previous bulk stores read the area
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 16 * pw.w + (pw.lane >> 2) + 8 * i;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = 8 * j + 2 * t;  // thread-owned 8-byte pieces: conflict-free per quarter-warp in the 128-B swizzle
        float2* dst = reinterpret_cast<float2*>(pw.stage + (c >> 5) * kBoxBytes + r * 128 +
                                                ((((c & 31) >> 2) ^ (r & 7)) << 4) + (c & 3) * 4);
        float2 v = make_float2(acc[0][4 * j + 2 * i], acc[0][4 * j + 2 * i + 1]);
        if (p.residual) { const float2 o = *dst; v.x += o.x; v.y += o.y; }
        if (p.bias) { v.x += bv[j].x; v.y += bv[j].y; }
        *dst = v;
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA unit
    named_bar_sync(GG_BAR_EPI + pw.wg, 128);                       // whole unit staged
    if (pw.w == 0 && pw.lane == 0) {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (n0 + 32 * c < p.N) tma_store_2d(&p.tmC, pw.stage_s + c * kBoxBytes, n0 + 32 * c, m0);
      tma_store_commit();
    }
  }
};
constexpr int UNIT_SMEM_TOTAL = pingpong_smem<UNIT_M, Fp32StagedEpilogue>();
static_assert(UNIT_SMEM_TOTAL <= 227 * 1024, "the 64-row ping-pong launch exceeds the 227 KB of shared memory per block");

__global__ void __launch_bounds__(GG_THREADS, 1) gemm_bf16_geglu_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                        const __grid_constant__ CUtensorMap tmB,
                                                                        const __grid_constant__ EpiParams p) {
  gemm_pingpong<false, 128>(tmA, tmB, p, tmA, tmB, p, GegluEpilogue{});
}

// ---------------------------------------------------------------------------------------------------
// gemm_bf16_kernel<EPI, DUAL>: the fp32 single-problem instance runs the ping-pong body on 64-row units, the bf16 ones
// the quadrant body, the two-problem ones (epilogues 0 and 3) the ping-pong body on 128-row tiles
// ---------------------------------------------------------------------------------------------------
template <int EPI, bool DUAL>
__global__ void __launch_bounds__(DUAL || EPI == 0 ? GG_THREADS : GTHREADS, 1) gemm_bf16_kernel(
    const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ EpiParams p,
    const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
    const __grid_constant__ EpiParams p2) {
  if constexpr (DUAL) {
    static_assert(EPI == 0 || EPI == 3, "two-problem launches have the fp32 (+bias) or the q/k,v epilogue");
    if constexpr (EPI == 3) gemm_pingpong<true, 128>(tmA, tmB, p, tmA2, tmB2, p2, QkNormEpilogue{});
    else gemm_pingpong<true, 128>(tmA, tmB, p, tmA2, tmB2, p2, Fp32Epilogue<false>{});
  } else if constexpr (EPI == 0) {
    gemm_pingpong<false, UNIT_M>(tmA, tmB, p, tmA, tmB, p, Fp32StagedEpilogue{});
  } else {
    gemm_quadrant<EPI>(tmA, tmB, p);
  }
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

// fp32 [rows, cols] output, row pitch ld floats; box = [UNIT_M rows, 32 floats = 128 B], SWIZZLE_128B (TMA epilogue)
static int get_c_map(const void* ptr, int64_t rows, int64_t cols, int64_t ld, CUtensorMap* out) {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  static std::mutex mu;
  const MapKey key{ptr, rows, cols, ld, UNIT_M};
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end()) { *out = it->second; return 0; }
  EncodeTiledFn fn = encode_fn();
  PHK_REQUIRE(fn, PHK_E_UNSUPPORTED, "cuTensorMapEncodeTiled not available from the driver");
  const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {32, (cuuint32_t)UNIT_M};
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
  constexpr int threads = EPI == 0 ? GG_THREADS : GTHREADS;
  constexpr int smem = EPI == 0 ? UNIT_SMEM_TOTAL : SMEM_TOTAL;
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(gemm_bf16_kernel<EPI, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    mark_configured(&configured_mask);
  }
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = tiles < kNumSMs ? tiles : kNumSMs;
  PHK_CUDA(launch_pdl(gemm_bf16_kernel<EPI, false>, dim3(grid), dim3(threads), (size_t)smem, st, ta, tb, p, ta, tb, p));
  PHK_LAUNCH_CHECK();
  return 0;
}

static int launch_gemm_geglu(const CUtensorMap& ta, const CUtensorMap& tb, const EpiParams& p, cudaStream_t st) {
  static unsigned long long configured_mask = 0;
  if (!device_configured(&configured_mask)) {
    PHK_CUDA(cudaFuncSetAttribute(gemm_bf16_geglu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GG_SMEM_TOTAL));
    mark_configured(&configured_mask);
  }
  const int tiles = p.m_tiles * p.n_tiles;
  const int grid = tiles < kNumSMs ? tiles : kNumSMs;
  PHK_CUDA(launch_pdl(gemm_bf16_geglu_kernel, dim3(grid), dim3(GG_THREADS), (size_t)GG_SMEM_TOTAL, st, ta, tb, p));
  PHK_LAUNCH_CHECK();
  return 0;
}

template <int EPI>
static int launch_gemm_dual(const CUtensorMap& ta, const CUtensorMap& tb, const EpiParams& p, const CUtensorMap& ta2,
                            const CUtensorMap& tb2, const EpiParams& p2, cudaStream_t st) {
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(gemm_bf16_kernel<EPI, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GG_SMEM_TOTAL));
    mark_configured(&configured_mask);
  }
  const int tiles = p.m_tiles * p.n_tiles + p2.m_tiles * p2.n_tiles;
  const int grid = tiles < kNumSMs ? tiles : kNumSMs;
  PHK_CUDA(launch_pdl(gemm_bf16_kernel<EPI, true>, dim3(grid), dim3(GG_THREADS), (size_t)GG_SMEM_TOTAL, st, ta, tb, p, ta2, tb2, p2));
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
  const int um = epilogue == 0 ? UNIT_M : GM;  // rows of a work unit: the fp32 epilogue runs on 64-row units
  CUtensorMap ta, tb;
  PHK_TRY(get_tensor_map(A, M, K, lda, um, &ta));
  cudaStream_t st = to_stream(s);
  PHK_TRY(get_tensor_map(W, N, K, ldw, GN, &tb));
  EpiParams p{C, ldc, M, N, K, bias, residual, seg_len, seg_stride, seg_off, (int)((M + um - 1) / um), (N + GN - 1) / GN};
  PHK_REQUIRE((int64_t)p.m_tiles * p.n_tiles < (1LL << 31), PHK_E_UNSUPPORTED, "phk_gemm_bf16: too many tiles");
  PHK_TRY(maybe_tma_epilogue(p, epilogue));
  if (epilogue == 2) return launch_gemm_geglu(ta, tb, p, st);
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
  // (the two-problem launch stores from the accumulator registers: no TMA epilogue)
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
