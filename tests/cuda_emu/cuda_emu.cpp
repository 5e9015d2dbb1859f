// TEST INFRASTRUCTURE: fiber scheduler of cuda_emu.h.  The kernels themselves are the product's sources (csrc/train.cu,
// rowops.cu, gemm_simt.cu, attention.cu) compiled by g++; the only stand-in is the wgmma GEMM (tensor cores cannot be
// emulated thread by thread), stated below from its include/phk.h contract.
#include "cuda_emu.h"
#include <setjmp.h>
#if defined(__SANITIZE_ADDRESS__)  // PHK_EMU_ASAN=1 build: tell AddressSanitizer about the fiber stacks
#include <sanitizer/common_interface_defs.h>
#define EMU_ASAN_START(save, bottom, size) __sanitizer_start_switch_fiber(save, bottom, size)
#define EMU_ASAN_FINISH(save, bottom, size) __sanitizer_finish_switch_fiber(save, bottom, size)
#else
#define EMU_ASAN_START(save, bottom, size) do { } while (0)
#define EMU_ASAN_FINISH(save, bottom, size) do { } while (0)
#endif

namespace emu {
State S;
namespace {
// A fiber is ENTERED through its ucontext (fresh stack) and afterwards switched with _setjmp / _longjmp: glibc's
// swapcontext saves the signal mask with a system call on every switch, which made the scheduler 4x slower.
struct Fiber {
  ucontext_t ctx;
  jmp_buf jb;
  bool started = false;
  bool done = false;
  unsigned tid = 0;
  void* asan_fake = nullptr;
};
jmp_buf sched_jb;
void* sched_fake = nullptr;
const void* sched_bottom = nullptr;
size_t sched_size = 0;
constexpr size_t kStack = 128 * 1024;
std::vector<Fiber> fibers;
std::vector<char> stacks;
int cur = -1;
Group g_block;
std::vector<Group> g_warps;
std::vector<float> xchg;
const std::function<void()>* g_body = nullptr;
std::vector<char> dyn;

unsigned long events = 0;  // barrier releases + fiber exits: no event in a whole scheduler round = deadlock
void on_exit_group(Group& g) {
  g.alive -= 1;
  if (g.alive > 0 && g.count == g.alive) { g.count = 0; g.gen += 1; }
}
void trampoline() {
  EMU_ASAN_FINISH(nullptr, &sched_bottom, &sched_size);
  (*g_body)();
  Fiber& f = fibers[cur];
  f.done = true;
  events += 1;
  on_exit_group(g_block);
  on_exit_group(g_warps[f.tid >> 5]);
  EMU_ASAN_START(nullptr, sched_bottom, sched_size);
  _longjmp(sched_jb, 1);
}
}  // namespace

void yield() {
  Fiber& f = fibers[cur];
  EMU_ASAN_START(&f.asan_fake, sched_bottom, sched_size);
  if (!_setjmp(f.jb)) _longjmp(sched_jb, 1);
  EMU_ASAN_FINISH(f.asan_fake, &sched_bottom, &sched_size);
}
void barrier(Group& g) {
  const unsigned gen = g.gen;
  g.count += 1;
  if (g.count == g.alive) { g.count = 0; g.gen += 1; events += 1; return; }
  while (g.gen == gen) yield();
}
Group& block_group() { return g_block; }
Group& warp_group() { return g_warps[fibers[cur].tid >> 5]; }
float* warp_xchg() { return xchg.data() + (size_t)(fibers[cur].tid >> 5) * 32; }

// PHK_EMU_SHUFFLE=<seed>: blocks run in a random order and, inside a block, the runnable threads are resumed in a fresh
// random order every scheduler round.  The default (in-order) schedule would hide a missing __syncthreads() or an
// assumption about block order; the tests run both.
static uint64_t g_rng = 0;
static bool g_shuffle = false;
static uint64_t next_rand() {
  g_rng ^= g_rng << 13; g_rng ^= g_rng >> 7; g_rng ^= g_rng << 17;
  return g_rng;
}
static void set_shuffle(uint64_t seed) {
  g_shuffle = seed != 0;
  g_rng = 0x9E3779B97F4A7C15ull ^ (seed * 0x100000001b3ull);
  if (!g_rng) g_rng = 1;
}
static void init_schedule() {
  static bool done = false;
  if (done) return;
  done = true;
  const char* e = getenv("PHK_EMU_SHUFFLE");
  if (e && *e) set_shuffle((uint64_t)strtoull(e, nullptr, 10));
}
template <typename T> static void shuffle(std::vector<T>& v) {
  for (size_t i = v.size(); i > 1; --i) std::swap(v[i - 1], v[next_rand() % i]);
}

void set_schedule_seed(uint64_t seed) { init_schedule(); set_shuffle(seed); }

// ---- stream capture: a graph is the list of operations submitted between Begin and End, replayed in order ----------
struct Graph { std::vector<std::function<void()>> nodes; };
static Graph* g_capturing = nullptr;
void submit(std::function<void()> op) {
  if (g_capturing) g_capturing->nodes.push_back(std::move(op));
  else op();
}

void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body) {
  init_schedule();
  const unsigned nt = block.x * block.y * block.z;
  if (block.y != 1 || block.z != 1) { fprintf(stderr, "cuda_emu: only 1-D blocks\n"); abort(); }
  if (fibers.size() < nt) { fibers.resize(nt); stacks.resize((size_t)nt * kStack); }
  dyn.assign(smem + 16, 0);
  const unsigned nw = (nt + 31) / 32;
  std::vector<uint64_t> order((size_t)grid.x * grid.y * grid.z);
  for (size_t i = 0; i < order.size(); ++i) order[i] = i;
  if (g_shuffle) shuffle(order);
  std::vector<unsigned> tids(nt);
  for (uint64_t lin : order) {
        const unsigned bx = (unsigned)(lin % grid.x), by = (unsigned)((lin / grid.x) % grid.y), bz = (unsigned)(lin / ((uint64_t)grid.x * grid.y));
        g_body = &body;
        g_block = Group{(int)nt, 0, 0};
        g_warps.assign(nw, Group{});
        for (unsigned w = 0; w < nw; ++w) g_warps[w].alive = (int)((w + 1) * 32 <= nt ? 32 : nt - w * 32);
        xchg.assign((size_t)nw * 32, 0.f);
        for (unsigned t = 0; t < nt; ++t) {
          Fiber& f = fibers[t];
          f.done = false; f.started = false; f.tid = t;
          getcontext(&f.ctx);
          f.ctx.uc_stack.ss_sp = stacks.data() + (size_t)t * kStack;
          f.ctx.uc_stack.ss_size = kStack;
          f.ctx.uc_link = nullptr;
          makecontext(&f.ctx, trampoline, 0);
        }
        unsigned remaining = nt;
        while (remaining) {
          const unsigned long before = events;
          for (unsigned t = 0; t < nt; ++t) tids[t] = t;
          if (g_shuffle) shuffle(tids);
          for (unsigned ti = 0; ti < nt; ++ti) {
            const unsigned t = tids[ti];
            Fiber& f = fibers[t];
            if (f.done) continue;
            cur = (int)t;
            S.t_idx = dim3(t, 0, 0); S.b_idx = dim3(bx, by, bz); S.b_dim = block; S.g_dim = grid;
            S.dyn_smem = dyn.data();
            EMU_ASAN_START(&sched_fake, stacks.data() + (size_t)t * kStack, kStack);
            if (!_setjmp(sched_jb)) {
              if (f.started) _longjmp(f.jb, 1);
              f.started = true;
              setcontext(&f.ctx);
            }
            EMU_ASAN_FINISH(sched_fake, nullptr, nullptr);
            if (f.done) { remaining -= 1; }
          }
          if (events == before) { fprintf(stderr, "cuda_emu: deadlock (a barrier some threads never reach)\n"); abort(); }
        }
      }
}
}  // namespace emu

cudaError_t cudaStreamBeginCapture(cudaStream_t, int) {
  if (emu::g_capturing) return cudaErrorInvalidValue;
  emu::g_capturing = new emu::Graph();
  return 0;
}
cudaError_t cudaStreamEndCapture(cudaStream_t, cudaGraph_t* g) {
  *g = emu::g_capturing;
  emu::g_capturing = nullptr;
  return *g ? 0 : cudaErrorInvalidValue;
}
cudaError_t cudaGraphInstantiate(cudaGraphExec_t* e, cudaGraph_t g, unsigned long long) {
  *e = new emu::Graph(*static_cast<emu::Graph*>(g));
  return 0;
}
static long g_graph_launches = 0;
cudaError_t cudaGraphLaunch(cudaGraphExec_t e, cudaStream_t) {
  g_graph_launches += 1;
  for (auto& op : static_cast<emu::Graph*>(e)->nodes) emu::submit(op);
  return 0;
}
extern "C" long phk_emu_graph_launches(void) { return g_graph_launches; }  // test hook
cudaError_t cudaGraphDestroy(cudaGraph_t g) { delete static_cast<emu::Graph*>(g); return 0; }
cudaError_t cudaGraphExecDestroy(cudaGraphExec_t e) { delete static_cast<emu::Graph*>(e); return 0; }

namespace phk {
// patchify_tma.cu (TMA) is not part of the emulated build: "shape not eligible" sends phk_patchify_ln to its plain kernels
int patchify_ln_tma_launch(const float*, int, int, int, int, int, int, int, int, int, int, const float*, const float*, void*,
                           int, cudaStream_t) { return 1; }
}  // namespace phk
// ---------------------------------------------------------------------------------------------------------------------
// The wgmma / TMA entry points (gemm_wgmma.cu, attention_tc.cu, head_sample.cu) cannot be executed thread by thread;
// they are represented by their include/phk.h CONTRACTS so that the bf16-mode drivers (weight packing, buffer wiring,
// the CFG-pair sharing, the masked-rows tail) can run end to end on the CPU.  Numerics: bf16 operands, fp32 accumulation.
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int phk_attention(const float*, const float*, const float*, const float*, const float*, const float*,
                             const uint8_t*, const float*, void*, const phk_attn_geom_t*, phk_stream_t);
extern "C" int phk_gemm_bf16(const void*, int64_t, const void*, int64_t, void*, int64_t, int64_t, int32_t, int32_t,
                             const float*, const float*, int64_t, int64_t, int64_t, int32_t, phk_stream_t);
extern "C" int phk_gemm_bf16_x2(const void* A1, int64_t lda1, const void* W1, int64_t ldw1, float* C1, int64_t ldc1,
                                int64_t M1, int32_t N1, int32_t K1, const float* bias1, const void* A2, int64_t lda2,
                                const void* W2, int64_t ldw2, float* C2, int64_t ldc2, int64_t M2, int32_t N2, int32_t K2,
                                const float* bias2, phk_stream_t s) {
  const int rc = phk_gemm_bf16(A1, lda1, W1, ldw1, C1, ldc1, M1, N1, K1, bias1, nullptr, 0, 0, 0, 0, s);
  return rc ? rc : phk_gemm_bf16(A2, lda2, W2, ldw2, C2, ldc2, M2, N2, K2, bias2, nullptr, 0, 0, 0, 0, s);
}
extern "C" int64_t phk_attention_tc_scratch_bytes(int32_t, int32_t, int32_t) { return 256; }
// q fp32 [n_seq*n, heads*64], kv fp32 [n_seq*n, 2*heads*64], bias [heads, n, n] -> out bf16: the fp32 kernel of the same
// contract (attention.cu) with bf16 output stands in (the real kernel also rounds q, k, v to bf16 first)
extern "C" int phk_attention_tc(const float* q, const float* kv, const float* q_scale, const float* k_scale,
                                const float* bias, void* out_bf16, int32_t n_seq, int32_t n, int32_t heads, float scale,
                                void*, int64_t, phk_stream_t s) {
  const int I = heads * 64;
  phk_attn_geom_t g;
  memset(&g, 0, sizeof(g));
  g.n_outer = n_seq; g.n_inner = 1; g.n_q = n; g.n_k = n; g.heads = heads; g.dim_head = 64;
  g.q_outer = (int64_t)n * I; g.q_tok = I; g.k_outer = (int64_t)n * 2 * I; g.k_tok = 2 * I; g.o_outer = g.q_outer; g.o_tok = I;
  g.mask_off_from = -1; g.out_bf16 = 1; g.scale = scale;
  return phk_attention(q, kv, nullptr, q_scale, k_scale, bias, nullptr, nullptr, out_bf16, &g, s);
}
// phk_attention_tc_bf16 contract: Qn [n_seq*n, ld_q] / KVn [n_seq*n, ld_kv] bf16, already normalised and scaled (the
// similarity scale folded into q); softmax(q k^T + bias) v per (sequence, head) -> out bf16 [n_seq*n, heads*64].  Like
// the kernel: fp32 scores / softmax statistics, probabilities rounded to bf16 before the P.V product.
extern "C" int phk_attention_tc_bf16(const void* Qn, int64_t ld_q, const void* KVn, int64_t ld_kv, const float* bias,
                                     void* out_bf16, int32_t n_seq, int32_t n, int32_t heads, phk_stream_t) {
  if (!Qn || !KVn || !out_bf16 || n_seq <= 0 || n <= 0 || heads <= 0) return PHK_E_ARG;
  emu::submit([=]() {
    const __nv_bfloat16* q = (const __nv_bfloat16*)Qn;
    const __nv_bfloat16* kv = (const __nv_bfloat16*)KVn;
    __nv_bfloat16* out = (__nv_bfloat16*)out_bf16;
    const int64_t I = (int64_t)heads * 64;
    std::vector<float> sc(n);
    for (int s_ = 0; s_ < n_seq; ++s_)
      for (int h = 0; h < heads; ++h)
        for (int i = 0; i < n; ++i) {
          const __nv_bfloat16* qi = q + ((int64_t)s_ * n + i) * ld_q + h * 64;
          float m = -INFINITY;
          for (int j = 0; j < n; ++j) {
            const __nv_bfloat16* kj = kv + ((int64_t)s_ * n + j) * ld_kv + h * 64;
            float a = 0.f;
            for (int d = 0; d < 64; ++d) a += __bfloat162float(qi[d]) * __bfloat162float(kj[d]);
            if (bias) a += bias[((int64_t)h * n + i) * n + j];
            sc[j] = a;
            m = fmaxf(m, a);
          }
          float sum = 0.f, o[64];
          for (int d = 0; d < 64; ++d) o[d] = 0.f;
          for (int j = 0; j < n; ++j) {
            const float e = expf(sc[j] - m);
            sum += e;
            const float eb = __bfloat162float(__float2bfloat16_rn(e));
            const __nv_bfloat16* vj = kv + ((int64_t)s_ * n + j) * ld_kv + I + h * 64;
            for (int d = 0; d < 64; ++d) o[d] += eb * __bfloat162float(vj[d]);
          }
          for (int d = 0; d < 64; ++d) out[((int64_t)s_ * n + i) * I + h * 64 + d] = __float2bfloat16_rn(o[d] / sum);
        }
  });
  return 0;
}
// phk_gemm_bf16_qkv contract: the q and k,v projections with the attention core's operands as output (bf16): per 64-column
// head l2-normalised (eps 1e-12) * learned scale (* sim_scale for q); the value half only converted
extern "C" int phk_gemm_bf16_qkv(const void* xn, const void* xraw, int64_t lda, const void* Wq, const void* Wkv, int64_t ldw,
                                 void* Qn, void* KVn, int64_t M, int32_t I, int32_t K, const float* q_scale,
                                 const float* k_scale, float sim_scale, phk_stream_t) {
  if (!xn || !xraw || !Wq || !Wkv || !Qn || !KVn || !q_scale || !k_scale || I % 128 || lda % 8 || ldw % 8) return PHK_E_ARG;
  emu::submit([=]() {
    auto project = [&](const void* A_, const void* W_, int N, int norm_cols, const float* scale, float mul, void* C_) {
      const __nv_bfloat16* a = (const __nv_bfloat16*)A_;
      const __nv_bfloat16* w = (const __nv_bfloat16*)W_;
      __nv_bfloat16* c = (__nv_bfloat16*)C_;
      std::vector<float> row(N);
      for (int64_t m = 0; m < M; ++m) {
        for (int nn = 0; nn < N; ++nn) {
          float acc = 0.f;
          for (int k = 0; k < K; ++k) acc += __bfloat162float(a[m * lda + k]) * __bfloat162float(w[(int64_t)nn * ldw + k]);
          row[nn] = acc;
        }
        for (int h0 = 0; h0 < N; h0 += 64) {
          if (h0 < norm_cols) {
            float ss = 0.f;
            for (int d = 0; d < 64; ++d) ss += row[h0 + d] * row[h0 + d];
            const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
            for (int d = 0; d < 64; ++d) c[m * N + h0 + d] = __float2bfloat16_rn((row[h0 + d] * inv) * (scale[d] * mul));
          } else {
            for (int d = 0; d < 64; ++d) c[m * N + h0 + d] = __float2bfloat16_rn(row[h0 + d]);
          }
        }
      }
    };
    project(xn, Wq, I, I, q_scale, sim_scale, Qn);
    project(xraw, Wkv, 2 * I, I, k_scale, 1.0f, KVn);
  });
  return 0;
}
// phk_layernorm_cfg / phk_head_sample (head_sample.cu, wgmma) from their include/phk.h contracts, for the drivers'
// wiring tests: e = s * norm(x_cond) + (1 - s) * norm(x_null) in bf16; logits = e W^T + bias in fp32, then the REAL
// phk_sample_tokens kernel (the documented equivalence: same Philox counter layout as phk_sample_tokens with u == NULL)
extern "C" int phk_layernorm_cfg(const float* xc, const float* xn, const float* g, const float* b, float scale, void* out,
                                 int64_t rows, int32_t dim, phk_stream_t) {
  emu::submit([=]() {
    __nv_bfloat16* o = (__nv_bfloat16*)out;
    std::vector<float> acc(dim);
    for (int64_t r = 0; r < rows; ++r) {
      for (int c = 0; c < dim; ++c) acc[c] = 0.f;
      for (int pass = 0; pass < 2; ++pass) {
        const float* x = (pass ? xn : xc) + r * dim;
        float mean = 0.f, var = 0.f;
        for (int c = 0; c < dim; ++c) mean += x[c];
        mean /= dim;
        for (int c = 0; c < dim; ++c) var += (x[c] - mean) * (x[c] - mean);
        const float rstd = 1.0f / sqrtf(var / dim + 1e-5f), w = pass ? 1.0f - scale : scale;
        for (int c = 0; c < dim; ++c) acc[c] += w * ((x[c] - mean) * rstd * g[c] + b[c]);
      }
      for (int c = 0; c < dim; ++c) o[r * dim + c] = __float2bfloat16_rn(acc[c]);
    }
  });
  return 0;
}
extern "C" int64_t phk_head_sample_scratch_bytes(int32_t n_tokens) { return (int64_t)n_tokens * 64 + 512; }
extern "C" int phk_sample_tokens(const float*, const float*, int64_t, const float*, uint64_t, uint64_t, float, float,
                                 const uint8_t*, int64_t*, int64_t*, float*, int64_t, int32_t, int64_t, int64_t, int64_t,
                                 phk_stream_t);
extern "C" int phk_head_sample_rng(const void* emb, int64_t ld_emb, int64_t emb_rows, const void* W, int64_t ldw,
                                   const float* bias, int32_t n_tokens, int32_t V, int32_t dim, float temperature,
                                   uint64_t seed, uint64_t offset, const uint64_t* rng_state, const uint8_t* mask,
                                   int64_t* ids, int64_t* pred_out, float* score_out, void*, int64_t, phk_stream_t s) {
  if (emb_rows < n_tokens || ld_emb % 8 || ldw % 8) return PHK_E_ARG;
  emu::submit([=]() {  // one stream-ordered operation; the device-resident noise key is read when it RUNS
    const __nv_bfloat16* e = (const __nv_bfloat16*)emb;
    const __nv_bfloat16* w = (const __nv_bfloat16*)W;
    std::vector<float> logits((size_t)n_tokens * V);
    for (int64_t r = 0; r < n_tokens; ++r)
      for (int v = 0; v < V; ++v) {
        float a = 0.f;
        for (int k = 0; k < dim; ++k) a += __bfloat162float(e[r * ld_emb + k]) * __bfloat162float(w[(int64_t)v * ldw + k]);
        logits[(size_t)r * V + v] = a + (bias ? bias[v] : 0.f);
      }
    const uint64_t sd = rng_state ? rng_state[0] : seed, of = rng_state ? rng_state[1] : offset;
    phk_sample_tokens(logits.data(), nullptr, V, nullptr, sd, of, 1.0f, temperature, mask, ids, pred_out, score_out, n_tokens,
                      V, 0, 0, 0, s);
  });
  return 0;
}
extern "C" int phk_head_sample(const void* emb, int64_t ld_emb, int64_t emb_rows, const void* W, int64_t ldw,
                               const float* bias, int32_t n_tokens, int32_t V, int32_t dim, float temperature, uint64_t seed,
                               uint64_t offset, const uint8_t* mask, int64_t* ids, int64_t* pred_out, float* score_out,
                               void* sc, int64_t sb, phk_stream_t s) {
  return phk_head_sample_rng(emb, ld_emb, emb_rows, W, ldw, bias, n_tokens, V, dim, temperature, seed, offset, nullptr, mask,
                             ids, pred_out, score_out, sc, sb, s);
}
// test hook: 0 = in-order schedule, otherwise the seed of the random block / thread order
extern "C" void phk_emu_set_shuffle(uint64_t seed) { emu::set_schedule_seed(seed); }

// wgmma GEMM contract (include/phk.h): bf16 operands K-major, fp32 accumulate; epilogue 0 fp32 (+bias, +residual, row
// map), 1 bf16 (+bias), 2 GEGLU over [64 value | 64 gate] row groups of W -> bf16 [M, N/2]
extern "C" int phk_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc, int64_t M,
                             int32_t N, int32_t K, const float* bias, const float* residual, int64_t seg_len,
                             int64_t seg_stride, int64_t seg_off, int32_t epilogue, phk_stream_t) {
  if (epilogue < 0 || epilogue > 2 || lda % 8 || ldw % 8 || lda < K || ldw < K) return PHK_E_ARG;
  if (epilogue == 2 && (N % 128 || bias || residual)) return PHK_E_ARG;
  emu::submit([=]() {
  const __nv_bfloat16* a = (const __nv_bfloat16*)A;
  const __nv_bfloat16* w = (const __nv_bfloat16*)W;
  std::vector<float> ar(K);
  auto dot = [&](int n) {
    float acc = 0.f;
    const __nv_bfloat16* wr = w + (int64_t)n * ldw;
    for (int k = 0; k < K; ++k) acc += ar[k] * __bfloat162float(wr[k]);
    return acc;
  };
  for (int64_t m = 0; m < M; ++m) {
    const int64_t orow = seg_len > 0 ? (m / seg_len) * seg_stride + seg_off + m % seg_len : m;
    for (int k = 0; k < K; ++k) ar[k] = __bfloat162float(a[m * lda + k]);
    if (epilogue == 2) {
      __nv_bfloat16* o = (__nv_bfloat16*)C;
      for (int t = 0; t < N / 128; ++t)
        for (int j = 0; j < 64; ++j) {
          const float val = dot(t * 128 + j), gate = dot(t * 128 + 64 + j);
          o[orow * ldc + t * 64 + j] = __float2bfloat16_rn(0.5f * gate * (1.0f + erff(gate * 0.70710678118654752440f)) * val);
        }
      continue;
    }
    for (int n = 0; n < N; ++n) {
      float acc = dot(n);
      if (bias) acc += bias[n];
      if (epilogue == 0) {
        float* c = (float*)C;
        if (residual) acc += residual[orow * ldc + n];
        c[orow * ldc + n] = acc;
      } else {
        ((__nv_bfloat16*)C)[orow * ldc + n] = __float2bfloat16_rn(acc);
      }
    }
  }
  });
  return 0;
}
