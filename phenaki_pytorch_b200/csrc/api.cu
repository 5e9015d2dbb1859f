// Fused drivers: the reference-facing operations as stream-ordered launch sequences.
//   phk_cvivit_encode     = CViViT.forward(video, return_only_codebook_ids=True)  cvivit.py:518-574
//   phk_maskgit_forward   = MaskGit.forward / TokenCritic.forward (CFG pair)      phenaki_pytorch.py:163-213, 265-302
// No host synchronisation, no allocation: scratch is carved from the caller's workspace.
#include "phk_common.cuh"
#include <atomic>
#include <cstring>
#include <cstdio>
#include <mutex>
#include <unordered_map>
#include <vector>

namespace phk {

static thread_local char g_err[256] = "";
static std::atomic<int64_t> g_launches{0};
void set_error(const char* msg) { std::snprintf(g_err, sizeof(g_err), "%s", msg); }
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

static std::atomic<int> g_prof_on{0};
struct ProfRec { int fam; cudaEvent_t e0, e1; double work; };
static std::vector<ProfRec> g_prof_recs;
static std::mutex g_prof_mu;
Prof::Prof(int f, phk_stream_t s, double w) : fam(f), st(to_stream(s)), e0(nullptr), on(false), work(w) {
  if (!g_prof_on.load(std::memory_order_relaxed)) return;
  on = true;
  cudaEventCreate(&e0);
  cudaEventRecord(e0, st);
}
Prof::~Prof() {
  if (!on) return;
  cudaEvent_t e1;
  cudaEventCreate(&e1);
  cudaEventRecord(e1, st);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_recs.push_back(ProfRec{fam, e0, e1, work});
}

// bump allocator over the caller's workspace (256-byte aligned slices)
struct Arena {
  char* base; int64_t size; int64_t off;
  void* take(int64_t bytes) {
    const int64_t o = (off + 255) & ~int64_t(255);
    off = o + bytes;
    return (off <= size && base) ? base + o : nullptr;
  }
};

struct SeqView {  // how sequences map onto rows of the [R, dim] residual stream
  int n_outer, n_inner, n_tok;
  int64_t outer, inner, tok;  // strides in ROWS
};

// Contraction type of one driver call + the PHK_PREC_BF16X3 split scratch (bf16 [rows, 3 * Kp] of the largest activation)
struct Lin { int prec; void* a3; int64_t a3_bytes; };
static inline int64_t x3_bytes(int64_t rows, int64_t Kmax) { return rows * 3 * ((Kmax + 7) / 8 * 8) * 2 + 256; }

struct TfCall {
  const phk_transformer_t* T;
  float* x;      // residual stream [R, dim] (in/out)
  float* x_alt;  // second buffer for the out-of-place PEG
  int64_t R;
  SeqView seq;
  int pegB, pegT, pegH, pegW, peg_layout;
  const float* attn_bias;      // [heads, n, n] or NULL
  const uint8_t* self_mask;    // [mask rows, n] or NULL
  int self_mask_mod;
  // cross attention
  const float* ctx_kv;         // [depth][ctx_rows][2I] pre-projected context keys/values, or NULL
  int ctx_b, ctx_L;            // context batch / length
  const uint8_t* ctx_mask;     // [ctx_b, L]
  int ctx_mask_off_from;       // sequences >= this see no text (CFG null half), -1: none
  int prec;
  Lin lin;                     // contraction type + split scratch of the nn.Linear products (prec is its .prec)
  void* out_cfg; float cfg_scale;  // bf16 [R/2, dim]: norm_out of the null half + scale * (cond - null) (fused head)
  // decoder tail: norm_out gathered into two dense operands (activation type of the mode) -- rows of the first
  // frame (t == 0) and of the remaining frames, each in (b,t,h,w) order (cvivit.py:506)
  void* out_first; void* out_rest; int split_B, split_T, split_hw;
  float** x_final;  // optional: receives the buffer holding the residual stream BEFORE norm_out (c.x or c.x_alt)
  // CFG pair (rows [0, R/2) conditional, [R/2, R) null) whose two halves enter with IDENTICAL rows: PEG and
  // self-attention of the first layer do not see the text, so they are computed for the first half only and copied
  // (the halves diverge at the first cross-attention).  Requires the n_inner == 1 sequence view.
  int dup_halves;
};

static int64_t tf_scratch_bytes(const phk_transformer_t* T, int64_t R) {
  const int64_t I = (int64_t)T->heads * T->dim_head;
  int64_t inner = 0;
  for (int l = 0; l < T->depth; ++l) inner = inner > T->layers[l].ff.inner ? inner : T->layers[l].ff.inner;
  // xn, q, kv, o, h(2*inner), g(inner)  -- all fp32 in parity mode
  // + head-major bf16 q/k/v^T operands of the tensor-core attention (bf16 mode): 3 * R * I * 2 bytes + padding
  return 256 * 14 + R * 4 * (T->dim + I + 2 * I + I + 2 * inner + inner) + R * I * 6 + 64 * 64 * 2 * (R / 64 + 64);
}

static int64_t tf_kmax(const phk_transformer_t* T) {  // largest K of a transformer's nn.Linear products
  int64_t k = T->dim > T->heads * T->dim_head ? T->dim : T->heads * T->dim_head;
  for (int l = 0; l < T->depth; ++l) k = k > T->layers[l].ff.inner ? k : T->layers[l].ff.inner;
  return k;
}
static inline bool known_prec(int prec) { return prec == PHK_PREC_F32 || prec == PHK_PREC_BF16 || prec == PHK_PREC_BF16X3; }

// y = act @ W^T (+bias)(+residual) in the selected contraction type.  `act` is fp32 (parity / split-bf16 modes) or bf16.
//   PHK_PREC_BF16X3: `act` fp32 is split into [hi | hi | lo] bf16 and multiplied with the [hi | lo | hi] weight pack
//   (w16, ld 3 * Kp) by ONE wgmma GEMM over K' = 3 Kp: fp32-grade products on the tensor cores.
static int linear(const Lin& ln, const void* act, int64_t lda, const float* w32, const void* w16, int64_t ldw, float* C,
                  int64_t ldc, int64_t M, int N, int K, const float* bias, const float* residual, phk_stream_t s) {
  if (ln.prec == PHK_PREC_BF16) {
    PHK_REQUIRE(w16, PHK_E_ARG, "bf16 mode needs the packed bf16 weight copies (*_h) in the weight table");
    return phk_gemm_bf16(act, lda, w16, ldw, C, ldc, M, N, K, bias, residual, 0, 0, 0, 0, s);
  }
  if (ln.prec == PHK_PREC_BF16X3) {
    PHK_REQUIRE(w16, PHK_E_ARG, "split-bf16 mode needs the [hi | lo | hi] weight packs (*_h) in the weight table");
    const int Kp = (K + 7) / 8 * 8;
    PHK_REQUIRE(ln.a3 && ln.a3_bytes >= M * 3 * (int64_t)Kp * 2, PHK_E_WORKSPACE, "split-bf16 mode: operand scratch too small");
    PHK_TRY(phk_split3((const float*)act, lda, ln.a3, M, K, 0, s));
    return phk_gemm_bf16(ln.a3, 3 * (int64_t)Kp, w16, 3 * (int64_t)Kp, C, ldc, M, N, 3 * Kp, bias, residual, 0, 0, 0, 0, s);
  }
  return phk_gemm_f32((const float*)act, lda, w32, ldw, C, ldc, M, N, K, bias, residual, 0, 0, 0, s);
}

// x <- Transformer(x)  (attention.py:311-332); the final norm_out is written to `out` (fp32) and, in bf16
// mode, optionally also to `out_h` (bf16, the A operand of a following head GEMM).
//   parity mode : every buffer fp32, FFMA GEMMs.
//   bf16 mode   : residual stream / LayerNorm / softmax fp32; LayerNorm emits bf16 GEMM operands (plus the
//                 un-normalised bf16 row for the self-attention k,v projection, attention.py:140-144); GEMMs on
//                 wgmma with fp32 accumulation; FF first linear fused with GEGLU; attention output bf16.
static int transformer_forward(const TfCall& c, Arena scratch, float* out, void* out_h, cudaStream_t st) {
  const phk_transformer_t* T = c.T;
  const bool h16 = c.prec == PHK_PREC_BF16;
  PHK_REQUIRE(c.prec == PHK_PREC_F32 || c.prec == PHK_PREC_BF16X3 || h16, PHK_E_ARG, "transformer: unknown precision mode");
  PHK_REQUIRE(c.lin.prec == c.prec, PHK_E_ARG, "transformer: contraction descriptor not initialised");
  const int D = T->dim, H = T->heads, DH = T->dim_head, I = H * DH;
  const int64_t R = c.R;
  int inner_max = 0;
  for (int l = 0; l < T->depth; ++l) inner_max = inner_max > T->layers[l].ff.inner ? inner_max : T->layers[l].ff.inner;
  const int64_t ab = h16 ? 2 : 4;  // activation bytes
  void* xn = scratch.take(R * D * ab);
  void* xraw = h16 ? scratch.take(R * D * 2) : nullptr;
  float* q = (float*)scratch.take(R * I * 4);
  float* kv = (float*)scratch.take(R * 2 * I * 4);
  void* o = scratch.take(R * I * ab);
  float* hbuf = h16 ? nullptr : (float*)scratch.take(R * 2 * (int64_t)inner_max * 4);
  void* gbuf = scratch.take(R * (int64_t)(h16 ? (inner_max + 63) / 64 * 64 * 2 : inner_max * 4));
  PHK_REQUIRE(xn && q && kv && o && gbuf && (h16 ? xraw != nullptr : hbuf != nullptr), PHK_E_WORKSPACE,
              "transformer: workspace too small");
  phk_stream_t s = reinterpret_cast<phk_stream_t>(st);
  float* x = c.x;
  float* x_alt = c.x_alt;

  // bf16 mode: cross-attention on packed operands -- the text keys / values of all layers are l2-normalised, scaled and
  // converted ONCE per call (phk_cross_kv_pack) instead of once per attention CTA, and the q projection's epilogue writes the
  // normalised bf16 queries (phk_gemm_bf16_qnorm): the attention kernel is 32 MMAs behind an 8 KB copy.
  void* cross_pack = nullptr;
  float* cross_dead = nullptr;
  int cross_nnull = 0;
#ifndef PHK_CUDA_EMU
  {
    bool ok = h16 && c.ctx_kv && DH == 64 && I % 128 == 0 && T->depth <= 16 && c.seq.n_inner == 1 && c.seq.tok == 1 &&
              c.seq.outer == c.seq.n_tok && c.ctx_b > 0;
    for (int l = 0; ok && l < T->depth; ++l) {
      const phk_layer_t& Ly = T->layers[l];
      ok = Ly.has_cross && Ly.cross_attn.wq_h && Ly.cross_attn.num_null_kv > 0 && Ly.cross_attn.null_kv &&
           Ly.cross_attn.num_null_kv == T->layers[0].cross_attn.num_null_kv &&
           Ly.cross_attn.num_null_kv + c.ctx_L <= 32;
    }
    if (ok) {
      Arena tmp = scratch;
      void* pk = tmp.take((int64_t)T->depth * c.ctx_b * H * 8192);
      float* dd = (float*)tmp.take((int64_t)T->depth * c.ctx_b * 32 * 4);
      if (pk && dd) {  // (a workspace sized by an older build: the unpacked kernel takes over)
        scratch = tmp;
        const float* kvp[16]; const float* nkp[16]; const float* ksp[16];
        for (int l = 0; l < T->depth; ++l) {
          kvp[l] = c.ctx_kv + (int64_t)l * c.ctx_b * c.ctx_L * 2 * I;
          nkp[l] = T->layers[l].cross_attn.null_kv;
          ksp[l] = T->layers[l].cross_attn.k_scale;
        }
        cross_nnull = T->layers[0].cross_attn.num_null_kv;
        PHK_TRY(phk_cross_kv_pack(kvp, nkp, ksp, T->depth, c.ctx_mask, c.ctx_b, c.ctx_L, H, cross_nnull, pk, dd, s));
        cross_pack = pk; cross_dead = dd;
      }
    }
  }
#endif
  for (int l = 0; l < T->depth; ++l) {
    const phk_layer_t& L = T->layers[l];
    // first layer of a CFG pair with identical halves: PEG + self-attention on the first half only
    const bool dup = l == 0 && c.dup_halves && c.seq.n_inner == 1 && c.seq.n_outer % 2 == 0 && c.pegB % 2 == 0 && R % 2 == 0;
    const int64_t Rl = dup ? R / 2 : R;
    const int n_outer = dup ? c.seq.n_outer / 2 : c.seq.n_outer;
    const int pegB = dup ? c.pegB / 2 : c.pegB;
    if (L.has_peg) {  // x = peg(x) + x
      PHK_REQUIRE((int64_t)pegB * c.pegT * c.pegH * c.pegW == Rl, PHK_E_SHAPE, "PEG: video shape does not cover the tokens");
      PHK_TRY(phk_peg3d(x, L.peg.w, L.peg.b, x_alt, pegB, c.pegT, c.pegH, c.pegW, D, L.peg.causal, c.peg_layout, s));
      float* t = x; x = x_alt; x_alt = t;
    }
    {  // x = self_attn(x) + x ; q from LN(x), k/v from RAW x (attention.py:140-144)
      const phk_attn_t& A = L.self_attn;
      PHK_TRY(phk_layernorm(x, A.norm_g, A.norm_b, xn, xraw, Rl, D, h16, 0, 0, 0, s));
      phk_attn_geom_t g;
      std::memset(&g, 0, sizeof(g));
      g.n_outer = n_outer; g.n_inner = c.seq.n_inner; g.n_q = c.seq.n_tok; g.n_k = c.seq.n_tok;
      g.heads = H; g.dim_head = DH; g.num_null_kv = A.num_null_kv; g.causal = T->causal;
      g.q_outer = c.seq.outer * I; g.q_inner = c.seq.inner * I; g.q_tok = c.seq.tok * I;
      g.k_outer = c.seq.outer * 2 * I; g.k_inner = c.seq.inner * 2 * I; g.k_tok = c.seq.tok * 2 * I;
      g.o_outer = g.q_outer; g.o_inner = g.q_inner; g.o_tok = g.q_tok;
      g.kv_outer_mod = 0; g.mask_outer_mod = c.self_mask_mod; g.mask_off_from = -1; g.out_bf16 = h16; g.scale = 8.f;
      const bool plain = h16 && DH == 64 && A.num_null_kv == 0 && !c.self_mask;
      const bool tc_ok = plain && !T->causal && c.seq.n_inner == 1 && c.seq.tok == 1 && c.seq.outer == c.seq.n_tok &&
                         c.seq.n_tok >= 64;
      const bool small_ok = plain && !c.attn_bias && c.seq.n_tok <= 16;
      // 16 < n <= 64 (the spatial transformer's 8 x 8 frames): warp-level MMAs, all (sequence, head) CTAs resident at once
      bool mid_ok = false;
#ifndef PHK_CUDA_EMU
      // (at exactly 64 tokens the wgmma kernel is used, so the MMA kernel takes 17..63 tokens)
      mid_ok = plain && !T->causal && c.seq.n_inner == 1 && c.seq.tok == 1 && c.seq.outer == c.seq.n_tok &&
               c.seq.n_tok > 16 && c.seq.n_tok < 64;
#endif
      if ((tc_ok || small_ok || mid_ok) && I % 128 == 0 && A.wq_h && A.wkv_h) {
        // q / k,v projections in ONE launch whose epilogue writes the attention core's bf16 operands directly
        // (l2-normalised q, k times their learned scales, the similarity scale 8 folded into q, v converted): no fp32
        // q / kv round trip and no separate normalisation pass (attention.py:146-157)
        void* qn = q;    // [Rl, I] bf16 in the fp32-sized q buffer
        void* kvn = kv;  // [Rl, 2I] bf16
        PHK_TRY(phk_gemm_bf16_qkv(xn, xraw, D, A.wq_h, A.wkv_h, D, qn, kvn, Rl, I, D, A.q_scale, A.k_scale, 8.f, s));
#ifndef PHK_CUDA_EMU
        if (mid_ok) PHK_TRY(phk_attention_mid_bf16(qn, I, kvn, 2 * I, c.attn_bias, o, n_outer, c.seq.n_tok, H, s));
        else
#endif
        if (tc_ok) PHK_TRY(phk_attention_tc_bf16(qn, I, kvn, 2 * I, c.attn_bias, o, n_outer, c.seq.n_tok, H, s));
        else PHK_TRY(phk_attention_small_bf16(qn, kvn, T->alibi_slopes, o, &g, s));
      } else {
        if (h16 && Rl > 128 && A.wq_h && A.wkv_h) {  // both projections in one launch (their tiles pipeline)
          PHK_TRY(phk_gemm_bf16_x2(xn, D, A.wq_h, D, q, I, Rl, I, D, nullptr, xraw, D, A.wkv_h, D, kv, 2 * I, Rl, 2 * I, D, nullptr, s));
        } else {
          PHK_TRY(linear(c.lin, xn, D, A.wq, A.wq_h, D, q, I, Rl, I, D, nullptr, nullptr, s));
          PHK_TRY(linear(c.lin, h16 ? xraw : (const void*)x, D, A.wkv, A.wkv_h, D, kv, 2 * I, Rl, 2 * I, D, nullptr, nullptr, s));
        }
        if (tc_ok) {  // wgmma path from fp32 projections (heads * 64 not a multiple of 128): operands prepared by attention_prep_kernel
          const int64_t ab = phk_attention_tc_scratch_bytes(n_outer, c.seq.n_tok, H);
          Arena tmp = scratch;
          void* asc = tmp.take(ab);
          PHK_REQUIRE(asc, PHK_E_WORKSPACE, "transformer: workspace too small (attention operands)");
          PHK_TRY(phk_attention_tc(q, kv, A.q_scale, A.k_scale, c.attn_bias, o, n_outer, c.seq.n_tok, H, 8.f, asc, ab, s));
        } else {
          PHK_TRY(phk_attention(q, kv, A.null_kv, A.q_scale, A.k_scale, c.attn_bias, c.self_mask, T->alibi_slopes, o, &g, s));
        }
      }
      PHK_TRY(linear(c.lin, o, I, A.wo, A.wo_h, I, x, D, Rl, D, I, nullptr, x, s));
    }
    if (dup)  // the null half continues from the same rows
      PHK_CUDA(cudaMemcpyAsync(x + Rl * D, x, Rl * D * 4, cudaMemcpyDeviceToDevice, st));
    if (L.has_cross && c.ctx_kv) {  // x = cross_attn(x, context) + x   (attention.py:327-328)
      const phk_attn_t& A = L.cross_attn;
      PHK_REQUIRE(c.seq.n_inner == 1, PHK_E_UNSUPPORTED, "cross attention needs (b, n) sequences");
      PHK_TRY(phk_layernorm(x, A.norm_g, A.norm_b, xn, nullptr, R, D, h16, 0, 0, 0, s));
#ifndef PHK_CUDA_EMU
      if (cross_pack) {
        PHK_TRY(phk_gemm_bf16_qnorm(xn, D, A.wq_h, D, q, R, I, D, A.q_scale, 8.f, s));  // bf16 [R, I] in the fp32-sized q buffer
        PHK_TRY(phk_attention_cross_packed(q, I, (char*)cross_pack + (int64_t)l * c.ctx_b * H * 8192,
                                           cross_dead + (int64_t)l * c.ctx_b * 32, o, I, c.seq.n_outer, c.seq.n_tok, H, c.ctx_b,
                                           cross_nnull, c.ctx_mask ? c.ctx_mask_off_from : -1, s));
      } else
#endif
      {
      PHK_TRY(linear(c.lin, xn, D, A.wq, A.wq_h, D, q, I, R, I, D, nullptr, nullptr, s));
      phk_attn_geom_t g;
      std::memset(&g, 0, sizeof(g));
      g.n_outer = c.seq.n_outer; g.n_inner = 1; g.n_q = c.seq.n_tok; g.n_k = c.ctx_L;
      g.heads = H; g.dim_head = DH; g.num_null_kv = A.num_null_kv; g.causal = 0;
      g.q_outer = c.seq.outer * I; g.q_inner = 0; g.q_tok = c.seq.tok * I;
      g.k_outer = (int64_t)c.ctx_L * 2 * I; g.k_inner = 0; g.k_tok = 2 * I;
      g.o_outer = g.q_outer; g.o_inner = 0; g.o_tok = g.q_tok;
      g.kv_outer_mod = c.ctx_b; g.mask_outer_mod = c.ctx_b; g.mask_off_from = c.ctx_mask_off_from;
      g.out_bf16 = h16; g.scale = 8.f;
      const float* kvl = c.ctx_kv + (int64_t)l * c.ctx_b * c.ctx_L * 2 * I;
      PHK_TRY(phk_attention(q, kvl, A.null_kv, A.q_scale, A.k_scale, nullptr, c.ctx_mask, nullptr, o, &g, s));
      }
      PHK_TRY(linear(c.lin, o, I, A.wo, A.wo_h, I, x, D, R, D, I, nullptr, x, s));
    }
    {  // x = ff(x) + x  (attention.py:45-53, 330)
      const phk_ff_t& Fw = L.ff;
      PHK_TRY(phk_layernorm(x, Fw.ln_g, Fw.ln_b, xn, nullptr, R, D, h16, 0, 0, 0, s));
      if (h16) {
        PHK_REQUIRE(Fw.w1_h && Fw.w2_h && Fw.inner_pad % 64 == 0 && Fw.inner_pad >= Fw.inner, PHK_E_ARG,
                    "bf16 mode needs the packed feed-forward weights");
        // first linear + GEGLU in one kernel (value/gate rows interleaved per 64), bf16 [R, inner_pad] out
        PHK_TRY(phk_gemm_bf16(xn, D, Fw.w1_h, D, gbuf, Fw.inner_pad, R, 2 * Fw.inner_pad, D, nullptr, nullptr, 0, 0, 0, 2, s));
        PHK_TRY(phk_gemm_bf16(gbuf, Fw.inner_pad, Fw.w2_h, Fw.inner_pad, x, D, R, D, Fw.inner_pad, nullptr, x, 0, 0, 0, 0, s));
      } else {
        PHK_TRY(linear(c.lin, xn, D, Fw.w1, Fw.w1_h, D, hbuf, 2 * Fw.inner, R, 2 * Fw.inner, D, nullptr, nullptr, s));
        PHK_TRY(phk_geglu(hbuf, (float*)gbuf, R, Fw.inner, s));
        PHK_TRY(linear(c.lin, gbuf, Fw.inner, Fw.w2, Fw.w2_h, Fw.inner, x, D, R, D, Fw.inner, nullptr, x, s));
      }
    }
  }
  if (c.x_final) *c.x_final = x;
  if (out) PHK_TRY(phk_layernorm(x, T->out_g, T->out_b, out, nullptr, R, D, 0, 0, 0, 0, s));
  if (c.out_cfg) {
    // classifier-free guidance folded before the (linear) logits head: rows [0,R/2) conditional, [R/2,R) null
    const int64_t half = R / 2;
    PHK_TRY(phk_layernorm_cfg(x, x + half * D, T->out_g, T->out_b, c.cfg_scale, c.out_cfg, half, D, s));
  }
  if (out_h) PHK_TRY(phk_layernorm(x, T->out_g, T->out_b, out_h, nullptr, R, D, 1, 0, 0, 0, s));
  if (c.out_first) {
    const int64_t hw = c.split_hw, per = (int64_t)c.split_T * hw;
    PHK_REQUIRE((int64_t)c.split_B * per == R, PHK_E_SHAPE, "transformer: frame split does not cover the tokens");
    PHK_TRY(phk_layernorm(x, T->out_g, T->out_b, c.out_first, nullptr, c.split_B * hw, D, h16, -hw, per, 0, s));
    if (c.split_T > 1) {
      PHK_REQUIRE(c.out_rest, PHK_E_ARG, "transformer: out_rest missing");
      PHK_TRY(phk_layernorm(x, T->out_g, T->out_b, c.out_rest, nullptr, c.split_B * (per - hw), D, h16, -(per - hw), per, hw, s));
    }
  }
  return 0;
}

static int check_transformer(const phk_transformer_t* T) {
  PHK_REQUIRE(T && T->layers && T->depth > 0 && T->dim > 0 && T->heads > 0 && T->dim_head > 0, PHK_E_ARG,
              "transformer table incomplete");
  PHK_REQUIRE(!T->causal || T->alibi_slopes, PHK_E_ARG, "causal transformer needs alibi_slopes");
  return 0;
}

}  // namespace phk

using namespace phk;

extern "C" int phk_version(void) { return 103; }
extern "C" const char* phk_last_error(void) { return g_err; }
extern "C" int64_t phk_launch_count(void) { return g_launches.load(); }

extern "C" int phk_prof_enable(int32_t on) { g_prof_on.store(on ? 1 : 0); return 0; }
// Sums the recorded per-call durations by kernel family (synchronises on the recorded events).
extern "C" int phk_prof_collect(double* ms_by_family, int64_t* calls_by_family, double* work_by_family, int32_t n) {
  PHK_REQUIRE(ms_by_family && calls_by_family && work_by_family && n >= FAM_COUNT, PHK_E_ARG, "phk_prof_collect: bad buffers");
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (int i = 0; i < n; ++i) { ms_by_family[i] = 0.0; calls_by_family[i] = 0; work_by_family[i] = 0.0; }
  for (auto& r : g_prof_recs) {
    PHK_CUDA(cudaEventSynchronize(r.e1));
    float ms = 0.f;
    PHK_CUDA(cudaEventElapsedTime(&ms, r.e0, r.e1));
    ms_by_family[r.fam] += ms; calls_by_family[r.fam] += 1; work_by_family[r.fam] += r.work;
    cudaEventDestroy(r.e0); cudaEventDestroy(r.e1);
  }
  g_prof_recs.clear();
  return 0;
}

// --------------------------------------------------------------------------------------------
// C-ViViT encode
// --------------------------------------------------------------------------------------------
static int cvivit_dims(const phk_cvivit_t* m, int32_t B, int32_t F, int& Tp, int& hh, int& ww, int64_t& R) {
  PHK_REQUIRE(m, PHK_E_ARG, "cvivit: null model");
  PHK_REQUIRE(B > 0 && F > 0, PHK_E_ARG, "cvivit: bad batch / frames");
  PHK_REQUIRE(m->patch_t > 0 && (F - 1) % m->patch_t == 0, PHK_E_SHAPE,
              "number of frames minus one must be divisible by temporal patch size (cvivit.py:540)");
  PHK_REQUIRE(m->image_h % m->patch_h == 0 && m->image_w % m->patch_w == 0, PHK_E_SHAPE,
              "image size must be divisible by patch size (cvivit.py:271)");
  Tp = 1 + (F - 1) / m->patch_t;
  hh = m->image_h / m->patch_h;
  ww = m->image_w / m->patch_w;
  R = (int64_t)B * Tp * hh * ww;
  return 0;
}

extern "C" int64_t phk_cvivit_workspace_bytes(const phk_cvivit_t* m, int32_t B, int32_t F, int32_t prec) {
  int Tp, hh, ww; int64_t R;
  if (cvivit_dims(m, B, F, Tp, hh, ww, R) != 0) return -1;
  const int64_t K2 = (int64_t)m->channels * m->patch_t * m->patch_h * m->patch_w;
  const int64_t hw = (int64_t)hh * ww;
  int64_t bytes = 256 * 16;
  bytes += R * K2 * 4;                 // patchified + normalised A operand (rest frames dominate)
  bytes += R * m->dim * 4 * 3;         // gemm out, x, x_alt
  bytes += (int64_t)m->heads * hw * hw * 4 + phk_cpb_scratch_floats(&m->spatial_bias, hh, ww, 1) * 4;
  const int64_t a = tf_scratch_bytes(&m->spatial, R), b = tf_scratch_bytes(&m->temporal, R);
  bytes += a > b ? a : b;
  if (m->codebook) bytes += phk_vq_cosine_scratch_bytes(R, m->codebook_size, prec == PHK_PREC_BF16 ? prec : PHK_PREC_F32) + 256;
  if (prec == PHK_PREC_BF16X3) {
    int64_t k = K2;
    k = k > tf_kmax(&m->spatial) ? k : tf_kmax(&m->spatial);
    k = k > tf_kmax(&m->temporal) ? k : tf_kmax(&m->temporal);
    bytes += x3_bytes(R, k);
  }
  return bytes;
}

static int cvivit_encode_impl(const phk_cvivit_t* m, const float* video, int32_t B, int32_t F, int64_t* ids,
                              void* workspace, int64_t workspace_bytes, int32_t prec, const float* spatial_bias,
                              float* tap_patch, float* tap_spatial, float* tap_temporal, float* tap_proj,
                              phk_stream_t s) {
  int Tp, hh, ww; int64_t R;
  PHK_TRY(cvivit_dims(m, B, F, Tp, hh, ww, R));
  PHK_REQUIRE(video && ids && workspace, PHK_E_ARG, "cvivit_encode: null pointer");
  PHK_TRY(check_transformer(&m->spatial));
  PHK_TRY(check_transformer(&m->temporal));
  PHK_REQUIRE(known_prec(prec), PHK_E_ARG, "cvivit_encode: unknown precision mode");
  const int h16 = prec == PHK_PREC_BF16;
  cudaStream_t st = to_stream(s);
  const int D = m->dim, hw = hh * ww;
  const int64_t K1 = (int64_t)m->channels * m->patch_h * m->patch_w, K2 = K1 * m->patch_t;
  Arena ar{(char*)workspace, workspace_bytes, 0};
  float* A = (float*)ar.take(R * K2 * 4);
  float* P = (float*)ar.take(R * D * 4);
  float* x = (float*)ar.take(R * D * 4);
  float* x_alt = (float*)ar.take(R * D * 4);
  float* bias_buf = (float*)ar.take((int64_t)m->heads * hw * hw * 4);
  float* cpb_scratch = (float*)ar.take(phk_cpb_scratch_floats(&m->spatial_bias, hh, ww, 1) * 4);
  PHK_REQUIRE(A && P && x && x_alt && bias_buf && cpb_scratch, PHK_E_WORKSPACE, "cvivit_encode: workspace too small");
  Lin lin{prec, nullptr, 0};
  if (prec == PHK_PREC_BF16X3) {
    int64_t k = K2;
    k = k > tf_kmax(&m->spatial) ? k : tf_kmax(&m->spatial);
    k = k > tf_kmax(&m->temporal) ? k : tf_kmax(&m->temporal);
    lin.a3_bytes = x3_bytes(R, k);
    lin.a3 = ar.take(lin.a3_bytes);
    PHK_REQUIRE(lin.a3, PHK_E_WORKSPACE, "cvivit_encode: workspace too small (split operands)");
  }

  // ---- to_patch_emb_first_frame / to_patch_emb (cvivit.py:542-549), rows land in (b,t,h,w) order
  const int C = m->channels, H = m->image_h, W = m->image_w;
  if (h16 && Tp > 1 && m->pf_w_h && m->pr_w_h) {
    // bf16 mode: both patch embeddings in ONE two-problem GEMM launch (16 + 128 tiles at cfg2: the first-frame
    // product alone occupied 16 SMs for 24 us).  A_rest at A, A_first behind it; outputs share P.
    const int64_t rows1 = (int64_t)B * hw, rows2 = (int64_t)B * (Tp - 1) * hw;
    char* A_first = (char*)A + ((rows2 * K2 * 2 + 255) / 256) * 256;
    PHK_REQUIRE((A_first - (char*)A) + rows1 * K1 * 2 <= R * K2 * 4, PHK_E_WORKSPACE, "cvivit_encode: workspace too small");
    PHK_TRY(phk_patchify_ln(video, B, C, F, H, W, 0, 1, 1, m->patch_h, m->patch_w, m->pf_ln1_g, m->pf_ln1_b, A_first, 1, s));
    PHK_TRY(phk_patchify_ln(video, B, C, F, H, W, 1, Tp - 1, m->patch_t, m->patch_h, m->patch_w, m->pr_ln1_g,
                            m->pr_ln1_b, A, 1, s));
    PHK_TRY(phk_gemm_bf16_x2(A_first, K1, m->pf_w_h, K1, P, D, rows1, D, (int)K1, m->pf_b, A, K2, m->pr_w_h, K2,
                             P + rows1 * D, D, rows2, D, (int)K2, m->pr_b, s));
    PHK_TRY(phk_layernorm(P, m->pf_ln2_g, m->pf_ln2_b, x, nullptr, rows1, D, 0, hw, (int64_t)Tp * hw, 0, s));
    PHK_TRY(phk_layernorm(P + rows1 * D, m->pr_ln2_g, m->pr_ln2_b, x, nullptr, rows2, D, 0, (int64_t)(Tp - 1) * hw,
                          (int64_t)Tp * hw, hw, s));
  } else {
  PHK_TRY(phk_patchify_ln(video, B, C, F, H, W, 0, 1, 1, m->patch_h, m->patch_w, m->pf_ln1_g, m->pf_ln1_b, A, h16, s));
  PHK_TRY(linear(lin, A, K1, m->pf_w, m->pf_w_h, K1, P, D, (int64_t)B * hw, D, (int)K1, m->pf_b, nullptr, s));
  PHK_TRY(phk_layernorm(P, m->pf_ln2_g, m->pf_ln2_b, x, nullptr, (int64_t)B * hw, D, 0, hw, (int64_t)Tp * hw, 0, s));
  if (Tp > 1) {
    const int64_t rows = (int64_t)B * (Tp - 1) * hw;
    PHK_TRY(phk_patchify_ln(video, B, C, F, H, W, 1, Tp - 1, m->patch_t, m->patch_h, m->patch_w, m->pr_ln1_g,
                            m->pr_ln1_b, A, h16, s));
    PHK_TRY(linear(lin, A, K2, m->pr_w, m->pr_w_h, K2, P, D, rows, D, (int)K2, m->pr_b, nullptr, s));
    PHK_TRY(phk_layernorm(P, m->pr_ln2_g, m->pr_ln2_b, x, nullptr, rows, D, 0, (int64_t)(Tp - 1) * hw,
                          (int64_t)Tp * hw, hw, s));
  }
  }
  if (tap_patch) PHK_CUDA(cudaMemcpyAsync(tap_patch, x, R * D * 4, cudaMemcpyDeviceToDevice, st));

  // ---- encode (cvivit.py:449-474): spatial over (b t), temporal over (b h w); no rearrange copies
  if (!spatial_bias) {
    PHK_TRY(phk_cpb_bias(&m->spatial_bias, hh, ww, 1, cpb_scratch, bias_buf, s));
    spatial_bias = bias_buf;
  }
  Arena tf = ar;
  TfCall c;
  std::memset(&c, 0, sizeof(c));
  c.T = &m->spatial; c.x = x; c.x_alt = x_alt; c.R = R;
  c.seq = SeqView{B * Tp, 1, hw, hw, 0, 1};
  c.pegB = B; c.pegT = Tp; c.pegH = hh; c.pegW = ww; c.peg_layout = 0;
  c.attn_bias = spatial_bias; c.ctx_mask_off_from = -1; c.prec = prec; c.lin = lin;
  PHK_TRY(transformer_forward(c, tf, P, nullptr, st));  // P <- norm_out(spatial)
  if (tap_spatial) PHK_CUDA(cudaMemcpyAsync(tap_spatial, P, R * D * 4, cudaMemcpyDeviceToDevice, st));

  c.T = &m->temporal; c.x = P; c.x_alt = x;
  c.seq = SeqView{B, hw, Tp, (int64_t)Tp * hw, 1, hw};
  c.peg_layout = 1;  // the reference's raw-reshape quirk (attention.py:71, cvivit.py:468-470)
  c.attn_bias = nullptr;
  // norm_out of the temporal transformer is fused with the LFQ projection + sign quantisation (cvivit.py:562-574):
  // the normalised tokens are only written when a parity test taps them; ids come out in (b, t, h, w) order
  float* xf = nullptr;
  c.x_final = &xf;
  PHK_TRY(transformer_forward(c, tf, nullptr, nullptr, st));
  float* norm_buf = x_alt;  // not used by the temporal transformer (its stream alternates between P and x)
  if (m->codebook) {
    // lookup_free_quantization=False (cvivit.py:321, 568-570): norm_out, then the nearest unit codebook row by cosine
    PHK_REQUIRE(m->codebook_size > 0, PHK_E_ARG, "cvivit_encode: codebook without a size");
    const int vprec = prec == PHK_PREC_BF16 ? prec : PHK_PREC_F32;  // (split-bf16 mode: the fp32 similarity path)
    const int64_t vb = phk_vq_cosine_scratch_bytes(R, m->codebook_size, vprec);
    void* vsc = tf.take(vb);
    PHK_REQUIRE(vsc, PHK_E_WORKSPACE, "cvivit_encode: workspace too small (codebook lookup)");
    if (tap_temporal || !h16) PHK_TRY(phk_layernorm(xf, m->temporal.out_g, m->temporal.out_b, norm_buf, nullptr, R, D, 0, 0, 0, 0, s));
    if (tap_temporal) PHK_CUDA(cudaMemcpyAsync(tap_temporal, norm_buf, R * D * 4, cudaMemcpyDeviceToDevice, st));
    if (h16) PHK_TRY(phk_layernorm(xf, m->temporal.out_g, m->temporal.out_b, norm_buf, nullptr, R, D, 1, 0, 0, 0, s));
    return phk_vq_cosine_ids(norm_buf, m->codebook, m->codebook_h, ids, R, D, m->codebook_size, vsc, vb, vprec, s);
  }
  PHK_TRY(phk_layernorm_lfq(xf, m->temporal.out_g, m->temporal.out_b, m->vq_w, m->vq_b, ids,
                            (tap_temporal || D % 128 != 0 || D > 1024 || m->codebook_bits > 16) ? norm_buf : nullptr,
                            tap_proj, R, D, m->codebook_bits, s));
  if (tap_temporal) PHK_CUDA(cudaMemcpyAsync(tap_temporal, norm_buf, R * D * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// ---- CUDA-graph replay of the encode --------------------------------------------------------------------------
// One encode is ~75 dependent launches of 3-40 us each; on a slow host the ~0.4-0.7 ms of launch calls per step is
// as long as the GPU work (0.85 ms in bf16 mode).  The launch sequence is a pure function of (weight table contents,
// buffers, shape, precision), so the second call with the same key captures it on a library-owned stream and later
// calls replay the instantiated graph on the caller's stream (one cudaGraphLaunch).  The first call always runs
// eagerly (one-time cudaFuncSetAttribute / tensor-map creation happen outside capture).  Disabled while the per-family
// profiler is on, when a parity test taps intermediates, and for good after a failed capture.
struct EncodeGraphKey {
  uint64_t table_hash;
  const void *video, *ids, *ws, *bias;
  int64_t ws_bytes;
  int B, F, prec, device;
  bool operator==(const EncodeGraphKey& o) const {
    return table_hash == o.table_hash && video == o.video && ids == o.ids && ws == o.ws && bias == o.bias &&
           ws_bytes == o.ws_bytes && B == o.B && F == o.F && prec == o.prec && device == o.device;
  }
};
struct EncodeGraphKeyHash {
  size_t operator()(const EncodeGraphKey& k) const {
    uint64_t h = k.table_hash;
    const uint64_t v[] = {(uint64_t)(uintptr_t)k.video, (uint64_t)(uintptr_t)k.ids, (uint64_t)(uintptr_t)k.ws,
                          (uint64_t)(uintptr_t)k.bias, (uint64_t)k.ws_bytes,
                          ((uint64_t)k.B << 40) ^ ((uint64_t)k.F << 20) ^ ((uint64_t)k.prec << 8) ^ (uint64_t)k.device};
    for (uint64_t x : v) h = (h ^ x) * 0x100000001b3ull;
    return (size_t)h;
  }
};
struct EncodeGraphEntry { cudaGraphExec_t exec; int launches; int seen; };

static uint64_t fnv(const void* p, size_t n, uint64_t h) {
  const unsigned char* c = (const unsigned char*)p;
  for (size_t i = 0; i < n; ++i) h = (h ^ c[i]) * 0x100000001b3ull;
  return h;
}
static uint64_t hash_transformer(const phk_transformer_t& T, uint64_t h) {
  h = fnv(&T, sizeof(T), h);
  if (T.layers && T.depth > 0) h = fnv(T.layers, sizeof(phk_layer_t) * (size_t)T.depth, h);
  return h;
}

extern "C" int phk_cvivit_encode(const phk_cvivit_t* m, const float* video, int32_t B, int32_t F, int64_t* ids,
                                 void* workspace, int64_t workspace_bytes, int32_t prec, const float* spatial_bias,
                                 float* tap_patch, float* tap_spatial, float* tap_temporal, float* tap_proj,
                                 phk_stream_t s) {
  const bool taps = tap_patch || tap_spatial || tap_temporal || tap_proj;
  if (!m || taps || !spatial_bias || g_prof_on.load(std::memory_order_relaxed))
    return cvivit_encode_impl(m, video, B, F, ids, workspace, workspace_bytes, prec, spatial_bias, tap_patch, tap_spatial,
                              tap_temporal, tap_proj, s);
  static std::unordered_map<EncodeGraphKey, EncodeGraphEntry, EncodeGraphKeyHash> cache;
  static std::mutex mu;
  static cudaStream_t cap = nullptr;
  static bool broken = false;  // a capture failed once: stay on the eager path
  int dev = 0;
  PHK_CUDA(cudaGetDevice(&dev));
  uint64_t th = fnv(m, sizeof(*m), 0xcbf29ce484222325ull);
  th = hash_transformer(m->spatial, th);
  th = hash_transformer(m->temporal, th);
  const EncodeGraphKey key{th, video, ids, workspace, spatial_bias, workspace_bytes, B, F, prec, dev};
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end() && it->second.exec) {
    PHK_CUDA(cudaGraphLaunch(it->second.exec, to_stream(s)));
    count_launch(it->second.launches);
    return 0;
  }
  if (broken || it == cache.end()) {  // first sighting of this key (or graphs unusable): run eagerly
    if (!broken) {
      if (cache.size() > 64) {  // bounded: drop everything (graphs are cheap to rebuild)
        for (auto& kv : cache) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
        cache.clear();
      }
      cache.emplace(key, EncodeGraphEntry{nullptr, 0, 1});
    }
    return cvivit_encode_impl(m, video, B, F, ids, workspace, workspace_bytes, prec, spatial_bias, nullptr, nullptr,
                              nullptr, nullptr, s);
  }
  // second sighting: capture on the library's stream, instantiate, replay on the caller's stream
  if (!cap) PHK_CUDA(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
  const int64_t l0 = g_launches.load();
  cudaGraph_t graph = nullptr;
  cudaError_t e = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
  int rc = 0;
  if (e == cudaSuccess) {
    rc = cvivit_encode_impl(m, video, B, F, ids, workspace, workspace_bytes, prec, spatial_bias, nullptr, nullptr, nullptr,
                            nullptr, reinterpret_cast<phk_stream_t>(cap));
    e = cudaStreamEndCapture(cap, &graph);
  }
  const int launches = (int)(g_launches.load() - l0);
  g_launches.store(l0);  // the captured launches did not execute
  cudaGraphExec_t exec = nullptr;
  if (e == cudaSuccess && rc == 0 && graph) e = cudaGraphInstantiate(&exec, graph, 0);
  if (graph) cudaGraphDestroy(graph);
  if (e != cudaSuccess || rc != 0 || !exec) {
    cudaGetLastError();  // clear the sticky capture error; fall back for good
    broken = true;
    return cvivit_encode_impl(m, video, B, F, ids, workspace, workspace_bytes, prec, spatial_bias, nullptr, nullptr,
                              nullptr, nullptr, s);
  }
  it->second.exec = exec;
  it->second.launches = launches;
  PHK_CUDA(cudaGraphLaunch(exec, to_stream(s)));
  count_launch(launches);
  return 0;
}

extern "C" int phk_cvivit_encode_host(const phk_cvivit_t* m, const float* host_video, int32_t B, int32_t F,
                                      int64_t* host_ids, void* dev_video, int64_t* dev_ids, void* workspace,
                                      int64_t workspace_bytes, int32_t prec, const float* spatial_bias,
                                      phk_stream_t s) {
  int Tp, hh, ww; int64_t R;
  PHK_TRY(cvivit_dims(m, B, F, Tp, hh, ww, R));
  PHK_REQUIRE(host_video && host_ids && dev_video && dev_ids, PHK_E_ARG, "cvivit_encode_host: null pointer");
  cudaStream_t st = to_stream(s);
  const int64_t vbytes = (int64_t)B * m->channels * F * m->image_h * m->image_w * 4;
  PHK_CUDA(cudaMemcpyAsync(dev_video, host_video, vbytes, cudaMemcpyHostToDevice, st));
  PHK_TRY(phk_cvivit_encode(m, (const float*)dev_video, B, F, dev_ids, workspace, workspace_bytes, prec, spatial_bias,
                            nullptr, nullptr, nullptr, nullptr, s));
  PHK_CUDA(cudaMemcpyAsync(host_ids, dev_ids, R * 8, cudaMemcpyDeviceToHost, st));
  PHK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// --------------------------------------------------------------------------------------------
// Host-buffer encode pipeline: the H2D copy of call i+1 (107 MB at cfg2, ~2 ms of PCIe) runs on the pipe's own copy
// stream while call i is still encoding on the caller's stream; the caller provides `depth` staging slots.
// --------------------------------------------------------------------------------------------
struct phk_encode_pipe {
  int depth;
  int64_t next;                          // next ticket
  cudaStream_t copy;
  std::vector<cudaEvent_t> h2d_done;     // [depth] copy stream: the slot's video has landed
  std::vector<cudaEvent_t> slot_free;    // [depth] compute stream: the encode that read the slot has finished
  std::vector<cudaEvent_t> done;         // [depth] compute stream: the slot's ids are in host memory
};

extern "C" int phk_encode_pipe_create(phk_encode_pipe_t** out, int32_t depth) {
  PHK_REQUIRE(out && depth >= 1 && depth <= 8, PHK_E_ARG, "phk_encode_pipe_create: depth must be 1..8");
  phk_encode_pipe* p = new phk_encode_pipe();
  p->depth = depth; p->next = 0; p->copy = nullptr;
  cudaError_t e = cudaStreamCreateWithFlags(&p->copy, cudaStreamNonBlocking);
  for (int i = 0; i < depth && e == cudaSuccess; ++i) {
    cudaEvent_t a = nullptr, b = nullptr, c = nullptr;
    e = cudaEventCreateWithFlags(&a, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&b, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c, cudaEventDisableTiming);
    p->h2d_done.push_back(a); p->slot_free.push_back(b); p->done.push_back(c);
  }
  if (e != cudaSuccess) { phk_encode_pipe_destroy(p); PHK_CUDA(e); }
  *out = p;
  return 0;
}

extern "C" int phk_encode_pipe_destroy(phk_encode_pipe_t* p) {
  if (!p) return 0;
  for (auto ev : p->h2d_done) if (ev) cudaEventDestroy(ev);
  for (auto ev : p->slot_free) if (ev) cudaEventDestroy(ev);
  for (auto ev : p->done) if (ev) cudaEventDestroy(ev);
  if (p->copy) cudaStreamDestroy(p->copy);
  delete p;
  return 0;
}

extern "C" int phk_encode_pipe_submit(phk_encode_pipe_t* p, const phk_cvivit_t* m, const float* host_video, int32_t B,
                                      int32_t F, int64_t* host_ids, void* dev_video_slots, int64_t* dev_ids_slots,
                                      void* workspace, int64_t workspace_bytes, int32_t prec,
                                      const float* spatial_bias, phk_stream_t s, int64_t* ticket) {
  int Tp, hh, ww; int64_t R;
  PHK_REQUIRE(p, PHK_E_ARG, "phk_encode_pipe_submit: null pipe");
  PHK_TRY(cvivit_dims(m, B, F, Tp, hh, ww, R));
  PHK_REQUIRE(host_video && host_ids && dev_video_slots && dev_ids_slots, PHK_E_ARG, "phk_encode_pipe_submit: null pointer");
  cudaStream_t st = to_stream(s);
  const int slot = (int)(p->next % p->depth);
  const int64_t vbytes = (int64_t)B * m->channels * F * m->image_h * m->image_w * 4;
  char* dv = (char*)dev_video_slots + (int64_t)slot * vbytes;
  int64_t* di = dev_ids_slots + (int64_t)slot * R;
  // the slot's previous occupant must have been consumed before it is overwritten (no-op for a fresh event)
  PHK_CUDA(cudaStreamWaitEvent(p->copy, p->slot_free[slot], 0));
  PHK_CUDA(cudaMemcpyAsync(dv, host_video, vbytes, cudaMemcpyHostToDevice, p->copy));
  PHK_CUDA(cudaEventRecord(p->h2d_done[slot], p->copy));
  PHK_CUDA(cudaStreamWaitEvent(st, p->h2d_done[slot], 0));
  PHK_TRY(phk_cvivit_encode(m, (const float*)dv, B, F, di, workspace, workspace_bytes, prec, spatial_bias, nullptr,
                            nullptr, nullptr, nullptr, s));
  PHK_CUDA(cudaEventRecord(p->slot_free[slot], st));
  PHK_CUDA(cudaMemcpyAsync(host_ids, di, R * 8, cudaMemcpyDeviceToHost, st));
  PHK_CUDA(cudaEventRecord(p->done[slot], st));
  if (ticket) *ticket = p->next;
  p->next += 1;
  return 0;
}

extern "C" int phk_encode_pipe_wait(phk_encode_pipe_t* p, int64_t ticket) {
  PHK_REQUIRE(p, PHK_E_ARG, "phk_encode_pipe_wait: null pipe");
  PHK_REQUIRE(ticket >= 0 && ticket < p->next && ticket >= p->next - p->depth, PHK_E_ARG,
              "phk_encode_pipe_wait: ticket is not in flight (already overwritten or never submitted)");
  PHK_CUDA(cudaEventSynchronize(p->done[(int)(ticket % p->depth)]));
  return 0;
}

// --------------------------------------------------------------------------------------------
// C-ViViT decode (cvivit.py:437-443, 476-516)
// --------------------------------------------------------------------------------------------
static int cvivit_dec_dims(const phk_cvivit_dec_t* m, int32_t B, int32_t Tp, int& hh, int& ww, int64_t& R) {
  PHK_REQUIRE(m, PHK_E_ARG, "cvivit_decode: null model");
  PHK_REQUIRE(B > 0 && Tp > 0, PHK_E_ARG, "cvivit_decode: bad batch / token-frame count");
  PHK_REQUIRE(m->patch_h > 0 && m->patch_w > 0 && m->patch_t > 0 && m->image_h % m->patch_h == 0 &&
              m->image_w % m->patch_w == 0, PHK_E_SHAPE, "image size must be divisible by patch size (cvivit.py:271)");
  hh = m->image_h / m->patch_h;
  ww = m->image_w / m->patch_w;
  R = (int64_t)B * Tp * hh * ww;
  return 0;
}

extern "C" int64_t phk_cvivit_decode_workspace_bytes(const phk_cvivit_dec_t* m, int32_t B, int32_t Tp, int32_t prec) {
  int hh, ww; int64_t R;
  if (cvivit_dec_dims(m, B, Tp, hh, ww, R) != 0) return -1;
  const int64_t hw = (int64_t)hh * ww, K1 = (int64_t)m->channels * m->patch_h * m->patch_w, K2 = K1 * m->patch_t;
  const int64_t g1 = (int64_t)B * hw * K1, g2 = (int64_t)B * (Tp - 1) * hw * K2;
  int64_t bytes = 256 * 16;
  bytes += R * m->dim * 4 * 4;                       // x, x_alt, norm_out(temporal), gathered GEMM operands
  bytes += (g1 > g2 ? g1 : g2) * 4;                  // to_pixels output before the un-patchify scatter
  bytes += (int64_t)m->heads * hw * hw * 4 + phk_cpb_scratch_floats(&m->spatial_bias, hh, ww, 1) * 4;
  const int64_t a = tf_scratch_bytes(&m->spatial, R), b = tf_scratch_bytes(&m->temporal, R);
  bytes += a > b ? a : b;
  if (prec == PHK_PREC_BF16X3) bytes += x3_bytes(R, tf_kmax(&m->spatial) > tf_kmax(&m->temporal) ? tf_kmax(&m->spatial) : tf_kmax(&m->temporal));
  return bytes;
}

extern "C" int phk_cvivit_decode(const phk_cvivit_dec_t* m, const int64_t* ids, const float* tokens, int32_t B,
                                 int32_t Tp, float* video, void* workspace, int64_t workspace_bytes, int32_t prec,
                                 const float* spatial_bias, float* tap_codes, float* tap_temporal,
                                 float* tap_spatial, phk_stream_t s) {
  int hh, ww; int64_t R;
  PHK_TRY(cvivit_dec_dims(m, B, Tp, hh, ww, R));
  PHK_REQUIRE((ids || tokens) && video && workspace, PHK_E_ARG, "cvivit_decode: null pointer");
  PHK_TRY(check_transformer(&m->spatial));
  PHK_TRY(check_transformer(&m->temporal));
  PHK_REQUIRE(known_prec(prec), PHK_E_ARG, "cvivit_decode: unknown precision mode");
  const int h16 = prec == PHK_PREC_BF16;
  cudaStream_t st = to_stream(s);
  const int D = m->dim, hw = hh * ww, C = m->channels;
  const int64_t K1 = (int64_t)C * m->patch_h * m->patch_w, K2 = K1 * m->patch_t;
  const int64_t rows1 = (int64_t)B * hw, rows2 = (int64_t)B * (Tp - 1) * hw;
  const int F = 1 + (Tp - 1) * m->patch_t;
  const int64_t ab = h16 ? 2 : 4;
  Arena ar{(char*)workspace, workspace_bytes, 0};
  float* x = (float*)ar.take(R * D * 4);
  float* x_alt = (float*)ar.take(R * D * 4);
  float* P = (float*)ar.take(R * D * 4);
  char* Afirst = (char*)ar.take(rows1 * D * ab);
  char* Arest = (char*)ar.take((rows2 > 0 ? rows2 : 1) * D * ab);
  float* G = (float*)ar.take((rows1 * K1 > rows2 * K2 ? rows1 * K1 : rows2 * K2) * 4);
  float* bias_buf = (float*)ar.take((int64_t)m->heads * hw * hw * 4);
  float* cpb_scratch = (float*)ar.take(phk_cpb_scratch_floats(&m->spatial_bias, hh, ww, 1) * 4);
  PHK_REQUIRE(x && x_alt && P && Afirst && Arest && G && bias_buf && cpb_scratch, PHK_E_WORKSPACE,
              "cvivit_decode: workspace too small");
  Lin lin{prec, nullptr, 0};
  if (prec == PHK_PREC_BF16X3) {
    lin.a3_bytes = x3_bytes(R, tf_kmax(&m->spatial) > tf_kmax(&m->temporal) ? tf_kmax(&m->spatial) : tf_kmax(&m->temporal));
    lin.a3 = ar.take(lin.a3_bytes);
    PHK_REQUIRE(lin.a3, PHK_E_WORKSPACE, "cvivit_decode: workspace too small (split operands)");
  }

  // ---- codes = vq.indices_to_codes(ids) (cvivit.py:437-439), rows in (b,t,h,w) order
  if (ids) PHK_TRY(phk_lfq_codes(ids, m->vq_out_w, m->vq_out_b, x, R, D, m->codebook_bits, s));
  else PHK_CUDA(cudaMemcpyAsync(x, tokens, R * D * 4, cudaMemcpyDeviceToDevice, st));
  if (tap_codes) PHK_CUDA(cudaMemcpyAsync(tap_codes, x, R * D * 4, cudaMemcpyDeviceToDevice, st));

  // ---- decode (cvivit.py:476-502): temporal over (b h w), then spatial over (b t)
  Arena tf = ar;
  TfCall c;
  std::memset(&c, 0, sizeof(c));
  c.T = &m->temporal; c.x = x; c.x_alt = x_alt; c.R = R;
  c.seq = SeqView{B, hw, Tp, (int64_t)Tp * hw, 1, hw};
  c.pegB = B; c.pegT = Tp; c.pegH = hh; c.pegW = ww;
  c.peg_layout = 1;  // same raw-reshape quirk as the encoder (attention.py:71, cvivit.py:489-491)
  c.ctx_mask_off_from = -1; c.prec = prec; c.lin = lin;
  PHK_TRY(transformer_forward(c, tf, P, nullptr, st));  // P <- norm_out(temporal)
  if (tap_temporal) PHK_CUDA(cudaMemcpyAsync(tap_temporal, P, R * D * 4, cudaMemcpyDeviceToDevice, st));

  if (!spatial_bias) {
    PHK_TRY(phk_cpb_bias(&m->spatial_bias, hh, ww, 1, cpb_scratch, bias_buf, s));
    spatial_bias = bias_buf;
  }
  c.T = &m->spatial; c.x = P; c.x_alt = x;
  c.seq = SeqView{B * Tp, 1, hw, hw, 0, 1};
  c.peg_layout = 0;
  c.attn_bias = spatial_bias;
  c.out_first = Afirst; c.out_rest = Arest; c.split_B = B; c.split_T = Tp; c.split_hw = hw;
  PHK_TRY(transformer_forward(c, tf, tap_spatial, nullptr, st));

  // ---- to_pixels_first_frame / to_pixels (cvivit.py:506-514): Linear + un-patchify scatter
  PHK_TRY(linear(lin, Afirst, D, m->px_first_w, m->px_first_w_h, D, G, K1, rows1, (int)K1, D, m->px_first_b, nullptr, s));
  PHK_TRY(phk_unpatchify(G, K1, video, B, C, F, m->image_h, m->image_w, 0, 1, 1, m->patch_h, m->patch_w, s));
  if (Tp > 1) {
    PHK_TRY(linear(lin, Arest, D, m->px_w, m->px_w_h, D, G, K2, rows2, (int)K2, D, m->px_b, nullptr, s));
    PHK_TRY(phk_unpatchify(G, K2, video, B, C, F, m->image_h, m->image_w, 1, Tp - 1, m->patch_t, m->patch_h,
                           m->patch_w, s));
  }
  return 0;
}

// --------------------------------------------------------------------------------------------
// MaskGit / TokenCritic forward
// --------------------------------------------------------------------------------------------
extern "C" int64_t phk_maskgit_workspace_bytes(const phk_maskgit_t* m, int32_t b, int32_t n, int32_t L,
                                               int32_t cfg_pair, int32_t prec) {
  if (!m || b <= 0 || n <= 0) return -1;
  const int64_t R = (int64_t)b * n * (cfg_pair ? 2 : 1);
  int64_t bytes = 256 * 16 + R * m->dim * 4 * 3;
  bytes += tf_scratch_bytes(&m->transformer, R);
  if (m->has_bias) bytes += (int64_t)m->heads * n * n * 4 + (int64_t)8 * n * 8 * m->heads * 4 + (1 << 20);
  if (prec == PHK_PREC_BF16X3) bytes += x3_bytes(R, tf_kmax(&m->transformer));
  // packed cross-attention operands of every layer (phk_cross_kv_pack): 8 KB per (layer, text, head) + the dead-key flags
  bytes += (int64_t)m->transformer.depth * b * m->transformer.heads * 8192 + (int64_t)m->transformer.depth * b * 128 + 512;
  (void)L;
  return bytes;
}

// context_norm + to_kv of every cross-attention layer (attention.py:137-144): depends only on the text,
// so Phenaki.sample computes it once per call instead of once per forward (36x per 18-step sample).
// out_kv: [depth, b*L, 2I] fp32.  scratch: b*L*dim_context floats.
extern "C" int phk_maskgit_context_kv(const phk_maskgit_t* m, const float* context, int32_t b, int32_t L,
                                      float* out_kv, float* scratch, int32_t prec, phk_stream_t s) {
  PHK_REQUIRE(m && context && out_kv && scratch, PHK_E_ARG, "maskgit_context_kv: null pointer");
  PHK_REQUIRE(b > 0 && L > 0, PHK_E_ARG, "maskgit_context_kv: bad size");
  PHK_REQUIRE(known_prec(prec), PHK_E_ARG, "maskgit_context_kv: unknown precision mode");
  const int h16 = prec == PHK_PREC_BF16;
  const phk_transformer_t* T = &m->transformer;
  PHK_TRY(check_transformer(T));
  const int I = T->heads * T->dim_head;
  const int64_t rows = (int64_t)b * L;
  // split-bf16 mode: the [hi | hi | lo] copy of the normalised text rows lives behind them in `scratch` (3x floats)
  Lin lin{prec, nullptr, 0};
  if (prec == PHK_PREC_BF16X3 && T->depth > 0) {
    const int64_t dc = T->layers[0].cross_attn.dim_context;
    lin.a3 = reinterpret_cast<char*>(scratch) + ((rows * dc * 4 + 255) / 256) * 256;
    lin.a3_bytes = rows * dc * 8 - 256;  // what is left of the 3 * rows * dc floats the caller provides
  }
  for (int l = 0; l < T->depth; ++l) {
    const phk_layer_t& Ly = T->layers[l];
    PHK_REQUIRE(Ly.has_cross, PHK_E_SHAPE, "maskgit_context_kv: layer has no cross attention");
    const phk_attn_t& A = Ly.cross_attn;
    PHK_TRY(phk_layernorm(context, A.ctx_g, A.ctx_b, scratch, nullptr, rows, A.dim_context, h16, 0, 0, 0, s));
    PHK_TRY(linear(lin, scratch, A.dim_context, A.wkv, A.wkv_h, A.dim_context, out_kv + (int64_t)l * rows * 2 * I, 2 * I,
                   rows, 2 * I, A.dim_context, nullptr, nullptr, s));
  }
  return 0;
}

extern "C" int phk_maskgit_forward(const phk_maskgit_t* m, const int64_t* ids, int32_t b, int32_t n, int32_t pt,
                                   int32_t ph, int32_t pw, const float* ctx_kv, int32_t L, const uint8_t* text_mask,
                                   const uint8_t* video_mask, int32_t cfg_pair, int32_t return_embeds,
                                   const float* pos_bias, float* out, void* workspace, int64_t workspace_bytes,
                                   int32_t prec, phk_stream_t s) {
  PHK_REQUIRE(m && ids && out && workspace, PHK_E_ARG, "maskgit_forward: null pointer");
  PHK_REQUIRE(b > 0 && n > 0, PHK_E_ARG, "maskgit_forward: bad size");
  PHK_REQUIRE((int64_t)pt * ph * pw == n, PHK_E_SHAPE, "video patch shape must cover the token sequence");
  PHK_REQUIRE(n <= m->max_seq_len, PHK_E_SHAPE,
              "the video token sequence length is greater than max_seq_len (phenaki_pytorch.py:196)");
  PHK_REQUIRE(known_prec(prec), PHK_E_ARG, "maskgit_forward: unknown precision mode");
  const int h16 = prec == PHK_PREC_BF16;
  PHK_REQUIRE(!ctx_kv || text_mask, PHK_E_ARG, "maskgit_forward: context without text mask");
  const phk_transformer_t* T = &m->transformer;
  PHK_TRY(check_transformer(T));
  cudaStream_t st = to_stream(s);
  const int reps = cfg_pair ? 2 : 1;
  const int D = m->dim;
  const int64_t R = (int64_t)b * n * reps;
  Arena ar{(char*)workspace, workspace_bytes, 0};
  float* x = (float*)ar.take(R * D * 4);
  float* x_alt = (float*)ar.take(R * D * 4);
  float* emb = (float*)ar.take(R * D * 4);
  PHK_REQUIRE(x && x_alt && emb, PHK_E_WORKSPACE, "maskgit_forward: workspace too small");
  Lin lin{prec, nullptr, 0};
  if (prec == PHK_PREC_BF16X3) {
    lin.a3_bytes = x3_bytes(R, tf_kmax(T));
    lin.a3 = ar.take(lin.a3_bytes);
    PHK_REQUIRE(lin.a3, PHK_E_WORKSPACE, "maskgit_forward: workspace too small (split operands)");
  }
  if (m->has_bias && !pos_bias) {
    float* bias_buf = (float*)ar.take((int64_t)m->heads * n * n * 4);
    float* sc = (float*)ar.take(phk_cpb_scratch_floats(&m->pos_bias, pt, ph, pw) * 4);
    PHK_REQUIRE(bias_buf && sc, PHK_E_WORKSPACE, "maskgit_forward: workspace too small (bias)");
    PHK_TRY(phk_cpb_bias(&m->pos_bias, pt, ph, pw, sc, bias_buf, s));
    pos_bias = bias_buf;
  }
  PHK_TRY(phk_token_embed(ids, m->token_emb, m->pos_emb, x, b, n, D, m->num_tokens + 1,
                          m->is_critic ? -1.f : m->shrink_alpha, reps, s));
  TfCall c;
  std::memset(&c, 0, sizeof(c));
  c.T = T; c.x = x; c.x_alt = x_alt; c.R = R;
  c.seq = SeqView{b * reps, 1, n, n, 0, 1};
  c.pegB = b * reps; c.pegT = pt; c.pegH = ph; c.pegW = pw; c.peg_layout = 0;
  c.attn_bias = m->has_bias ? pos_bias : nullptr;
  c.self_mask = video_mask; c.self_mask_mod = b;
  c.ctx_kv = ctx_kv; c.ctx_b = b; c.ctx_L = L; c.ctx_mask = text_mask;
  c.ctx_mask_off_from = cfg_pair ? b : -1;
  c.dup_halves = cfg_pair ? 1 : 0;  // phk_token_embed wrote the same embeddings for both halves
  c.prec = prec; c.lin = lin;
  if (return_embeds || m->is_critic) return transformer_forward(c, ar, out, nullptr, st);
  // to_logits (phenaki_pytorch.py:213): the final LayerNorm feeds the head GEMM directly (bf16 operand in bf16 mode)
  PHK_TRY(transformer_forward(c, ar, h16 ? nullptr : emb, h16 ? (void*)emb : nullptr, st));
  PHK_TRY(linear(lin, emb, D, m->head_w, m->head_w_h, D, out, m->num_tokens, R, m->num_tokens, D, m->head_b, nullptr, s));
  return 0;
}

// One demasking iteration's network half, fully fused for the sampling loop (phenaki_pytorch.py:493-509, 547-550):
// MaskGit forward for the CFG pair, then logits head + CFG + gumbel argmax + confidence in ONE GEMM kernel whose
// epilogue reduces over the vocabulary -- the (2b, n, V) logits are never written.  bf16 mode, cond_scale != 1; with a
// prime prefix the head runs on the sampled tokens only.
extern "C" int64_t phk_maskgit_sample_workspace_bytes(const phk_maskgit_t* m, int32_t b, int32_t n, int32_t L) {
  if (!m || b <= 0 || n <= 0) return -1;
  const int64_t tokens = (int64_t)b * n;
  // the masked-rows-only tail (phk_sample_tail) never needs more than the all-rows one: its largest case is k = n
  const int64_t tail = phk_sample_tail_scratch_bytes(b, n, m->dim);
  const int64_t full = tokens * m->dim * 2 + phk_head_sample_scratch_bytes((int32_t)tokens);
  // (+1 MB: the head's per-split partials of a few-row tail, at most 128 * 148 * 20 B, are not monotonic in k)
  return phk_maskgit_workspace_bytes(m, b, n, L, 1, PHK_PREC_BF16) + (tail > full ? tail : full) + (1 << 20);
}

static int sample_step_impl(const phk_maskgit_t* m, const int64_t* ids_in, int32_t b, int32_t n, int32_t pt,
                            int32_t ph, int32_t pw, const float* ctx_kv, int32_t L,
                            const uint8_t* text_mask, const float* pos_bias,
                            float cond_scale, float temperature, uint64_t seed, uint64_t offset, const uint64_t* rng_state,
                            const uint8_t* mask, int64_t* ids, int64_t* pred_out, float* score_out,
                            int32_t masked_per_seq, int32_t prime_len, void* workspace, int64_t workspace_bytes,
                            phk_stream_t s) {
  // n = prime_len + sampled tokens per sequence (phenaki_pytorch.py:493: the prime ids are prepended at every step);
  // mask / ids / pred_out / score_out cover the sampled tokens only
  PHK_REQUIRE(m && ids_in && workspace, PHK_E_ARG, "maskgit_sample_step: null pointer");
  PHK_REQUIRE(prime_len >= 0 && prime_len < n, PHK_E_ARG, "maskgit_sample_step: prime_len out of range");
  const int32_t n_new = n - prime_len;
  PHK_REQUIRE(masked_per_seq >= 0 && masked_per_seq <= n_new, PHK_E_ARG, "maskgit_sample_step: masked_per_seq out of range");
  PHK_REQUIRE(prime_len == 0 || (mask && ids && masked_per_seq > 0), PHK_E_ARG,
              "maskgit_sample_step: a primed step needs the mask, the ids and the masked-token count");
  PHK_REQUIRE(b > 0 && n > 0 && (int64_t)pt * ph * pw == n, PHK_E_SHAPE, "video patch shape must cover the token sequence");
  PHK_REQUIRE(n <= m->max_seq_len, PHK_E_SHAPE,
              "the video token sequence length is greater than max_seq_len (phenaki_pytorch.py:196)");
  PHK_REQUIRE(!m->is_critic && m->head_w_h && cond_scale != 1.0f && m->dim <= 512 && m->dim % 128 == 0, PHK_E_UNSUPPORTED,
              "maskgit_sample_step: needs a MaskGit table with bf16 weights, dim % 128 == 0, dim <= 512 and guidance");
  PHK_REQUIRE(!ctx_kv || text_mask, PHK_E_ARG, "maskgit_sample_step: context without text mask");
  PHK_REQUIRE(workspace_bytes >= phk_maskgit_sample_workspace_bytes(m, b, n, L), PHK_E_WORKSPACE,
              "maskgit_sample_step: workspace too small");
  const phk_transformer_t* T = &m->transformer;
  PHK_TRY(check_transformer(T));
  cudaStream_t st = to_stream(s);
  const int D = m->dim;
  const int64_t tokens = (int64_t)b * n, R = 2 * tokens;
  Arena ar{(char*)workspace, workspace_bytes, 0};
  float* x = (float*)ar.take(R * D * 4);
  float* x_alt = (float*)ar.take(R * D * 4);
  // masked rows only (phk_sample_tail) when the caller vouches for the per-sequence count and it saves work
  const bool compact = mask && ids && masked_per_seq > 0 && masked_per_seq < n;
  const int64_t hb = compact ? phk_sample_tail_scratch_bytes(b, masked_per_seq, D) : phk_head_sample_scratch_bytes((int32_t)tokens);
  void* emb_h = compact ? nullptr : ar.take(tokens * D * 2);
  void* hsc = ar.take(hb);
  PHK_REQUIRE(x && x_alt && (compact || emb_h) && hsc, PHK_E_WORKSPACE, "maskgit_sample_step: workspace too small");
  if (m->has_bias && !pos_bias) {
    float* bias_buf = (float*)ar.take((int64_t)m->heads * n * n * 4);
    float* sc = (float*)ar.take(phk_cpb_scratch_floats(&m->pos_bias, pt, ph, pw) * 4);
    PHK_REQUIRE(bias_buf && sc, PHK_E_WORKSPACE, "maskgit_sample_step: workspace too small (bias)");
    PHK_TRY(phk_cpb_bias(&m->pos_bias, pt, ph, pw, sc, bias_buf, s));
    pos_bias = bias_buf;
  }
  PHK_TRY(phk_token_embed(ids_in, m->token_emb, m->pos_emb, x, b, n, D, m->num_tokens + 1, m->shrink_alpha, 2, s));
  TfCall c;
  std::memset(&c, 0, sizeof(c));
  c.T = T; c.x = x; c.x_alt = x_alt; c.R = R;
  c.seq = SeqView{2 * b, 1, n, n, 0, 1};
  c.pegB = 2 * b; c.pegT = pt; c.pegH = ph; c.pegW = pw; c.peg_layout = 0;
  c.attn_bias = m->has_bias ? pos_bias : nullptr;
  c.ctx_kv = ctx_kv; c.ctx_b = b; c.ctx_L = L; c.ctx_mask = text_mask; c.ctx_mask_off_from = b;
  c.prec = PHK_PREC_BF16; c.lin = Lin{PHK_PREC_BF16, nullptr, 0}; c.out_cfg = emb_h; c.cfg_scale = cond_scale;
  c.dup_halves = 1;  // phk_token_embed wrote the same embeddings for both halves
  float* xf = nullptr;
  c.x_final = &xf;  // the residual stream before norm_out: rows [0, tokens) conditional, [tokens, 2 tokens) null
  PHK_TRY(transformer_forward(c, ar, nullptr, nullptr, st));
  if (compact)
    return phk_sample_tail_rows(xf, xf + tokens * D, T->out_g, T->out_b, cond_scale, m->head_w_h, D, m->head_b, b, n_new,
                                masked_per_seq, m->num_tokens, D, temperature, seed, offset, rng_state, mask, ids, pred_out,
                                score_out, n, prime_len, hsc, hb, s);
  return phk_head_sample_rng(emb_h, D, tokens, m->head_w_h, D, m->head_b, (int32_t)tokens, m->num_tokens, D, temperature,
                             seed, offset, rng_state, mask, ids, pred_out, score_out, hsc, hb, s);
}

// ids_in (b, n) = prime ids followed by the tokens being sampled (prime_len == 0: no prefix; prime_len > 0:
// Phenaki.sample(prime_frames=...), make_video's scene chains); mask / ids / pred_out / score_out (b, n - prime_len) cover
// the sampled tokens.
extern "C" int phk_maskgit_sample_step(const phk_maskgit_t* m, const int64_t* ids_in, int32_t b, int32_t n, int32_t pt,
                                       int32_t ph, int32_t pw, const float* ctx_kv, int32_t L, const uint8_t* text_mask,
                                       const float* pos_bias, float cond_scale, float temperature, uint64_t seed,
                                       uint64_t offset, const uint8_t* mask, int64_t* ids, int64_t* pred_out,
                                       float* score_out, int32_t masked_per_seq, int32_t prime_len, void* workspace,
                                       int64_t workspace_bytes, phk_stream_t s) {
  return sample_step_impl(m, ids_in, b, n, pt, ph, pw, ctx_kv, L, text_mask, pos_bias, cond_scale, temperature, seed,
                          offset, nullptr, mask, ids, pred_out, score_out, masked_per_seq, prime_len, workspace,
                          workspace_bytes, s);
}

// ---- one whole demasking iteration, optionally replayed as a CUDA graph ---------------------------------------------
// Everything that changes between calls lives in device memory (ids / mask / scores / pred are updated in place, the
// noise key is rng_state), so the launch sequence is a pure function of the arguments and a captured graph stays valid:
// same scheme as phk_cvivit_encode (first sighting of a key eager, second captured, then one cudaGraphLaunch).

// Philox counters one iteration reserves: one V-wide draw over all b*n sampled tokens, one more, rounded up to the
// multiple of 4 torch's generator offsets take.  phenaki.py:_noise_stride is the same formula on the host side.
static uint64_t noise_stride(int32_t b, int32_t n, int32_t V) {
  return ((uint64_t)b * (uint64_t)n * (uint64_t)((V + 3) / 4) + 1 + 3) / 4 * 4;
}

static std::atomic<bool> g_step_graph{true};
// tests: 1 replays phk_maskgit_demask_iteration as a CUDA graph, 0 keeps it eager, < 0 back to the default (on)
extern "C" int phk_debug_step_graph(int32_t on) { g_step_graph.store(on != 0); return 0; }

// Launch-sequence cache of phk_maskgit_demask_iteration: `key` identifies the call (table contents, every pointer and
// scalar), `run(stream)` issues the launches.  First sighting of a key: eager; second: captured; later: one cudaGraphLaunch.
template <typename Run>
static int replay_or_capture(uint64_t key, phk_stream_t s, Run&& run) {
  struct Entry { cudaGraphExec_t exec; int launches; };
  static std::unordered_map<uint64_t, Entry> cache;
  static std::mutex mu;
  static cudaStream_t cap = nullptr;
  static bool broken = false;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it != cache.end() && it->second.exec) {
    PHK_CUDA(cudaGraphLaunch(it->second.exec, to_stream(s)));
    count_launch(it->second.launches);
    return 0;
  }
  if (broken || it == cache.end()) {  // first sighting (or graphs unusable): eager
    if (!broken) {
      if (cache.size() > 1024) {
        for (auto& kv : cache) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
        cache.clear();
      }
      cache.emplace(key, Entry{nullptr, 0});
    }
    return run(s);
  }
  if (!cap) PHK_CUDA(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
  const int64_t l0 = g_launches.load();
  cudaGraph_t graph = nullptr;
  cudaError_t e = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
  int rc = 0;
  if (e == cudaSuccess) {
    rc = run(reinterpret_cast<phk_stream_t>(cap));
    e = cudaStreamEndCapture(cap, &graph);
  }
  const int launches = (int)(g_launches.load() - l0);
  g_launches.store(l0);  // the captured launches did not execute
  cudaGraphExec_t exec = nullptr;
  if (e == cudaSuccess && rc == 0 && graph) e = cudaGraphInstantiate(&exec, graph, 0);
  if (graph) cudaGraphDestroy(graph);
  if (e != cudaSuccess || rc != 0 || !exec) {
    cudaGetLastError();
    broken = true;
    return run(s);
  }
  it->second.exec = exec;
  it->second.launches = launches;
  PHK_CUDA(cudaGraphLaunch(exec, to_stream(s)));
  count_launch(launches);
  return 0;
}

// ---- the iteration of a sample (phenaki_pytorch.py:478-550; make_video's scenes) -------------------------------------
// token_in [b, prime_len + n]: the MaskGit / critic input -- the prime ids in the first prime_len columns (written once by
// the caller), the sampled tokens copied in by the call (prime_len == 0: token_in is `ids` itself).
//   [k_remask > 0: re-mask the k_remask lowest-confidence... (phk_topk_mask on `scores`)]
//   -> ids -> token_in -> MaskGit CFG pair + tail on the masked rows -> ids / pred / scores (logit confidence) in place
//   -> rng_state[1] += noise_stride(b, n, V)
//   -> unless `skip_critic`: ids -> token_in -> critic forward of the CFG pair (critic: a TokenCritic table; NULL: the
//      MaskGit's own embeddings, SelfCritic) -> scores = critic head with guidance + noise_K * (u - 0.5) * noise_mult  (:534-545)
extern "C" int64_t phk_maskgit_demask_iteration_workspace_bytes(const phk_maskgit_t* m, const phk_maskgit_t* critic,
                                                                int32_t b, int32_t n_total, int32_t L) {
  if (!m || b <= 0 || n_total <= 0) return -1;
  const int64_t a = phk_maskgit_sample_workspace_bytes(m, b, n_total, L);
  const int64_t c = phk_maskgit_workspace_bytes(critic ? critic : m, b, n_total, L, 1, PHK_PREC_BF16);
  return (a > c ? a : c) + 2 * (int64_t)b * n_total * m->dim * 4 + 512;
}

static int demask_iteration_impl(const phk_maskgit_t* m, const phk_maskgit_t* critic, const float* head_w,
                                 const float* head_b, int64_t* token_in, int64_t* ids, uint8_t* mask, float* scores,
                                 int64_t* pred, int32_t b, int32_t n, int32_t prime_len, int32_t pt, int32_t ph, int32_t pw,
                                 const float* ctx_kv, const float* critic_ctx_kv, int32_t L, const uint8_t* text_mask,
                                 const float* pos_bias, float cond_scale, float temperature, uint64_t* rng_state,
                                 int32_t k_remask, const float* critic_noise, float noise_K, float noise_mult,
                                 int32_t skip_critic, void* workspace, int64_t workspace_bytes, phk_stream_t s) {
  cudaStream_t st = to_stream(s);
  const int32_t nt = prime_len + n;
  const int64_t need = phk_maskgit_demask_iteration_workspace_bytes(m, critic, b, nt, L);
  PHK_REQUIRE(workspace_bytes >= need, PHK_E_WORKSPACE, "maskgit_demask_iteration: workspace too small");
  const int64_t emb_bytes = 2 * (int64_t)b * nt * m->dim * 4;
  float* emb = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + ((workspace_bytes - emb_bytes) & ~(int64_t)255));
  const int64_t body_bytes = reinterpret_cast<char*>(emb) - reinterpret_cast<char*>(workspace);
  auto ids_to_input = [&]() -> int {
    if (token_in == ids) return 0;
    PHK_CUDA(cudaMemcpy2DAsync(token_in + prime_len, (size_t)nt * 8, ids, (size_t)n * 8, (size_t)n * 8, (size_t)b,
                               cudaMemcpyDeviceToDevice, st));
    return 0;
  };
  if (k_remask > 0) PHK_TRY(phk_topk_mask(scores, b, n, k_remask, mask, ids, (int64_t)m->num_tokens, s));
  PHK_TRY(ids_to_input());
  PHK_TRY(sample_step_impl(m, token_in, b, nt, pt, ph, pw, ctx_kv, L, text_mask, pos_bias, cond_scale, temperature, 0, 0,
                           rng_state, mask, ids, pred, scores, k_remask > 0 ? k_remask : n, prime_len, workspace, body_bytes, s));
  PHK_TRY(phk_rng_advance(rng_state, noise_stride(b, n, m->num_tokens), s));
  if (skip_critic) return 0;
  PHK_TRY(ids_to_input());
  const phk_maskgit_t* net = critic ? critic : m;
  PHK_TRY(phk_maskgit_forward(net, token_in, b, nt, pt, ph, pw, critic ? critic_ctx_kv : ctx_kv, L,
                              (critic ? critic_ctx_kv : ctx_kv) ? text_mask : nullptr, nullptr, 1, 1,
                              net->has_bias ? pos_bias : nullptr, emb, workspace, body_bytes, PHK_PREC_BF16, s));
  const int64_t half = (int64_t)b * nt * m->dim;
  return phk_critic_scores(emb, emb + half, head_w, head_b, critic_noise, cond_scale, noise_K, noise_mult, scores,
                           (int64_t)b * n, m->dim, prime_len ? n : 0, prime_len ? nt : 0, prime_len ? prime_len : 0, s);
}

extern "C" int phk_maskgit_demask_iteration(const phk_maskgit_t* m, const phk_maskgit_t* critic, const float* head_w,
                                            const float* head_b, int64_t* token_in, int64_t* ids, uint8_t* mask,
                                            float* scores, int64_t* pred, int32_t b, int32_t n, int32_t prime_len,
                                            int32_t pt, int32_t ph, int32_t pw, const float* ctx_kv,
                                            const float* critic_ctx_kv, int32_t L, const uint8_t* text_mask,
                                            const float* pos_bias, float cond_scale, float temperature,
                                            uint64_t* rng_state, int32_t k_remask, const float* critic_noise,
                                            float noise_K, float noise_mult, int32_t skip_critic, void* workspace,
                                            int64_t workspace_bytes, phk_stream_t s) {
  PHK_REQUIRE(m && token_in && ids && mask && scores && pred && rng_state && workspace, PHK_E_ARG,
              "maskgit_demask_iteration: null pointer");
  PHK_REQUIRE(n > 0 && prime_len >= 0 && k_remask >= 0 && k_remask <= n, PHK_E_ARG,
              "maskgit_demask_iteration: prime_len / k_remask out of range");
  PHK_REQUIRE(prime_len > 0 || token_in == ids, PHK_E_ARG,
              "maskgit_demask_iteration: without a prime prefix the input buffer is the id buffer");
  PHK_REQUIRE(skip_critic || (head_w && head_b), PHK_E_ARG, "maskgit_demask_iteration: critic head missing");
  PHK_REQUIRE(!critic || (critic->is_critic && critic->dim == m->dim), PHK_E_ARG,
              "maskgit_demask_iteration: the critic table must be a TokenCritic of the MaskGit's width");
  auto run = [&](phk_stream_t st) {
    return demask_iteration_impl(m, critic, head_w, head_b, token_in, ids, mask, scores, pred, b, n, prime_len, pt, ph, pw,
                                 ctx_kv, critic_ctx_kv, L, text_mask, pos_bias, cond_scale, temperature, rng_state,
                                 k_remask, critic_noise, noise_K, noise_mult, skip_critic, workspace, workspace_bytes, st);
  };
  if (!g_step_graph.load(std::memory_order_relaxed) || !pos_bias || g_prof_on.load(std::memory_order_relaxed)) return run(s);
  int dev = 0;
  PHK_CUDA(cudaGetDevice(&dev));
  // key: table contents + every pointer and scalar of the call (a 64-bit FNV of them; the values behind the pointers
  // -- token state, noise key, weights -- are read at replay time)
  uint64_t key = fnv(m, sizeof(*m), 0xcbf29ce484222325ull);
  key = hash_transformer(m->transformer, key);
  if (critic) {
    key = fnv(critic, sizeof(*critic), key);
    key = hash_transformer(critic->transformer, key);
  }
  const void* ptrs[] = {head_w, head_b, token_in, ids, mask, scores, pred, ctx_kv, critic_ctx_kv, text_mask, pos_bias, rng_state,
                        critic_noise, workspace};
  key = fnv(ptrs, sizeof(ptrs), key);
  const int64_t ints[] = {b, n, prime_len, pt, ph, pw, L, k_remask, skip_critic, dev, workspace_bytes};
  key = fnv(ints, sizeof(ints), key);
  const float fl[] = {cond_scale, temperature, noise_K, noise_mult};
  key = fnv(fl, sizeof(fl), key);
  return replay_or_capture(key, s, run);
}
