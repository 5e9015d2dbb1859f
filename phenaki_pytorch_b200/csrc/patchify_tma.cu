// Patchify + LayerNorm(K) (cvivit.py:273-275 / 280-282) with the token gathered by the TMA unit.
//
// The video (B,C,F,H,W) fp32 is described to the TMA unit as a 5-D tensor; one token is the box
// (1, C, pt, p1, p2) whose dense shared-memory image is exactly the reference's feature order (c pt p1 p2).  Each
// persistent CTA double-buffers two tokens: while all threads normalise token j out of one buffer, a single elected
// thread has already issued the bulk copy of token j+1 into the other, so the only HBM-visible read of the encoder
// (107 MB at cfg2) keeps streaming instead of stalling on the two block-wide reductions of every token.  gamma / beta
// are staged once per CTA.  Falls back to patchify_ln_reg_kernel (rowops.cu) when the shape does not fit a box.
#include "phk_common.cuh"
#include "phk_sm90.cuh"
#include <mutex>
#include <unordered_map>

namespace phk {
namespace {


__global__ void __launch_bounds__(256, 2) patchify_ln_tma_kernel(const __grid_constant__ CUtensorMap tmV, int hh, int ww,
                                                                 int f0, int nt, int pt, int p1, int p2, int K,
                                                                 const float* __restrict__ g, const float* __restrict__ b,
                                                                 void* __restrict__ out, int out_bf16, int tokens) {
  pdl_trigger();
  extern __shared__ __align__(128) uint8_t smem_raw[];
  __shared__ float red[32];
  __shared__ __align__(8) unsigned long long bars[2];
  const int K4 = K >> 2;
  float4* stage0 = reinterpret_cast<float4*>(smem_raw);                  // [K] floats, token buffer 0
  float4* stage1 = stage0 + K4;                                          // token buffer 1
  float4* sg = stage1 + K4;                                              // gamma
  float4* sb = sg + K4;                                                  // beta
  const uint32_t bar0 = smem_u32(&bars[0]);
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmV) : "memory");
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < K4; i += blockDim.x) {
    sg[i] = __ldg(reinterpret_cast<const float4*>(g) + i);
    sb[i] = __ldg(reinterpret_cast<const float4*>(b) + i);
  }
  __syncthreads();
  pdl_wait();  // gamma / beta are weights; the video may be produced by the previous kernel
  auto issue = [&](int token, int s) {  // one elected thread: bulk copy of a token's (1, C, pt, p1, p2) box
    int tok = token;
    const int wi = tok % ww; tok /= ww;
    const int hi = tok % hh; tok /= hh;
    const int ti = tok % nt;
    const int bi = tok / nt;
    const uint32_t bar = bar0 + 8 * s;
    mbar_expect_tx(bar, (uint32_t)K * 4u);
    tma_load_5d(&tmV, bar, smem_u32(s ? stage1 : stage0), wi * p2, hi * p1, f0 + ti * pt, 0, bi);
  };
  int token = blockIdx.x;
  if (threadIdx.x == 0 && token < tokens) issue(token, 0);
  for (int it = 0; token < tokens; ++it, token += gridDim.x) {
    const int s = it & 1;
    const int next = token + gridDim.x;
    if (threadIdx.x == 0 && next < tokens) issue(next, s ^ 1);  // buffer s^1 was released by the barrier ending it-1
    mbar_wait(bar0 + 8 * s, (uint32_t)(it >> 1) & 1u);
    const float4* v = s ? stage1 : stage0;
    float sum = 0.f;
    for (int i = threadIdx.x; i < K4; i += blockDim.x) { const float4 t = v[i]; sum += (t.x + t.y) + (t.z + t.w); }
    const float mean = block_sum(sum, red) / (float)K;
    float q = 0.f;
    for (int i = threadIdx.x; i < K4; i += blockDim.x) {
      const float4 t = v[i];
      const float a = t.x - mean, bq = t.y - mean, c = t.z - mean, d = t.w - mean;
      q += (a * a + bq * bq) + (c * c + d * d);
    }
    const float rstd = rsqrtf(block_sum(q, red) / (float)K + 1e-5f);
    const int64_t orow = (int64_t)token * K;
    for (int i = threadIdx.x; i < K4; i += blockDim.x) {
      const float4 t = v[i], gg = sg[i], bb = sb[i];
      float4 o;
      o.x = (t.x - mean) * rstd * gg.x + bb.x;
      o.y = (t.y - mean) * rstd * gg.y + bb.y;
      o.z = (t.z - mean) * rstd * gg.z + bb.z;
      o.w = (t.w - mean) * rstd * gg.w + bb.w;
      if (out_bf16)
        reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + orow)[i] =
            make_uint2(pack_bf16x2(o.x, o.y), pack_bf16x2(o.z, o.w));
      else
        reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + orow)[i] = o;
    }
    __syncthreads();  // every thread is done with buffer s: the elected thread may refill it next iteration
  }
}


struct VKey {
  const void* ptr; int B, C, F, H, W, pt, p1, p2;
  bool operator==(const VKey& o) const {
    return ptr == o.ptr && B == o.B && C == o.C && F == o.F && H == o.H && W == o.W && pt == o.pt && p1 == o.p1 && p2 == o.p2;
  }
};
struct VKeyHash {
  size_t operator()(const VKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    for (int v : {k.B, k.C, k.F, k.H, k.W, k.pt, k.p1, k.p2}) h = h * 1000003u ^ (size_t)v;
    return h;
  }
};

}  // namespace

// returns 0 when launched, 1 when the shape is not eligible (caller falls back), >1 / <0 on errors
int patchify_ln_tma_launch(const float* video, int B, int C, int F, int H, int W, int f0, int nt, int pt, int p1, int p2,
                           const float* ln_g, const float* ln_b, void* out, int out_bf16, cudaStream_t st) {
  const int K = C * pt * p1 * p2;
  const size_t smem = (size_t)4 * K * sizeof(float);  // two token buffers + gamma + beta
  if (p2 % 4 != 0 || W % 4 != 0 || (K * 4) % 128 != 0 || p1 > 256 || p2 > 256 || pt > 256 || C > 256 || smem > 100 * 1024 ||
      ((reinterpret_cast<uintptr_t>(video) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(ln_g) |
        reinterpret_cast<uintptr_t>(ln_b)) & 15) != 0)
    return 1;
  EncodeTiledFn fn = encode_fn();
  if (!fn) return 1;
  static std::unordered_map<VKey, CUtensorMap, VKeyHash> cache;
  static std::mutex mu;
  CUtensorMap map;
  {
    const VKey key{video, B, C, F, H, W, pt, p1, p2};
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(key);
    if (it != cache.end()) {
      map = it->second;
    } else {
      const cuuint64_t gdim[5] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)F, (cuuint64_t)C, (cuuint64_t)B};
      const cuuint64_t gstride[4] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4, (cuuint64_t)F * H * W * 4,
                                     (cuuint64_t)C * F * H * W * 4};
      const cuuint32_t box[5] = {(cuuint32_t)p2, (cuuint32_t)p1, (cuuint32_t)pt, (cuuint32_t)C, 1};
      const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
      const CUresult r = fn(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(video), gdim, gstride, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return 1;  // unusual pitch / alignment: the register kernel handles it
      if (cache.size() > 1024) cache.clear();
      cache.emplace(key, map);
    }
  }
  static unsigned long long configured_mask = 0;
  const bool configured = device_configured(&configured_mask);
  if (!configured) {
    PHK_CUDA(cudaFuncSetAttribute(patchify_ln_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    mark_configured(&configured_mask);
  }
  const int tokens = B * nt * (H / p1) * (W / p2);
  const unsigned grid = (unsigned)(tokens < 2 * kNumSMs ? tokens : 2 * kNumSMs);
  PHK_CUDA(launch_pdl(patchify_ln_tma_kernel, dim3(grid), dim3(256), smem, st, map, H / p1, W / p2, f0, nt, pt, p1, p2, K,
                      ln_g, ln_b, out, out_bf16, tokens));
  return 0;
}

}  // namespace phk
