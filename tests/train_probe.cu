// Test-only entry points into the training step's products: the shipped csrc/train.cu compiled unchanged, followed by
// extern "C" wrappers around its internal functions (which live in an anonymous namespace and are not exported by
// libphk.so).  The wrappers hold no logic of their own; tests/train_probe.py builds this file into a separate library,
// for the GPU with nvcc and for the CPU executor of tests/cuda_emu with g++.
#include "../phenaki_pytorch_b200/csrc/train.cu"

// sgemm_batched: C[m, n] (+)= sum_k A(m, k) B(k, n) over a two-level batch (GemmBatch), fp32 or bf16 products
extern "C" int probe_sgemm_batched(const float* A, int64_t sam, int64_t sak, const float* B, int64_t sbk, int64_t sbn,
                                   float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, int32_t accumulate,
                                   int32_t count, int32_t div, int64_t a_outer, int64_t a_inner, int64_t b_outer,
                                   int64_t b_inner, int64_t c_outer, int64_t c_inner, int32_t k_total,
                                   int32_t bf16_products, phk_stream_t s) {
  const phk::GemmBatch gb{count, div, a_outer, a_inner, b_outer, b_inner, c_outer, c_inner, k_total};
  return phk::sgemm_batched(A, sam, sak, B, sbk, sbn, C, ldc, M, N, K, accumulate, gb, phk::to_stream(s), bf16_products != 0);
}

// op 0: linear_fwd(x, w -> y, bias, residual), 1: dgrad_p(dy, w -> dx, accumulate), 2: wgrad_p(dy, x -> dw);
// scratch holds the two operand buffers of `elems` bf16 each, back to back
extern "C" int probe_linear(int32_t op, int32_t prec, void* scratch, int64_t elems, const float* a, const float* b,
                            float* out, int64_t M, int64_t N, int64_t K, const float* bias, const float* residual,
                            int32_t accumulate, phk_stream_t s) {
  __nv_bfloat16* base = static_cast<__nv_bfloat16*>(scratch);
  const phk::TcScratch tc{base, base ? base + elems : nullptr, elems};
  if (op == 0) return phk::linear_fwd(prec, tc, a, b, out, M, N, K, bias, residual, s);
  if (op == 1) return phk::dgrad_p(prec, tc, a, b, out, M, N, K, accumulate, s);
  if (op == 2) return phk::wgrad_p(prec, tc, a, b, out, M, N, K, s);
  return PHK_E_ARG;
}

extern "C" int probe_attention_backward(const float* q, const float* kv, const phk_attn_t* A, const phk_attn_t* G,
                                        const float* bias, const uint8_t* key_mask, const float* dO, float* dq,
                                        float* dkv, float* dbias, int32_t b, int32_t H, int32_t n, int32_t m,
                                        int32_t nnull, int32_t dh, float* scratch, int32_t bf16_products,
                                        phk_stream_t s) {
  const phk::AttnBwdGeom g{b, H, n, m, nnull, dh};
  return phk::attention_backward(q, kv, *A, *G, bias, key_mask, dO, dq, dkv, dbias, g, scratch, phk::to_stream(s),
                                 bf16_products != 0, phk::DropSite{0.f, 1.f, 0, 0, 0});
}

// out[0..7]: float offsets of qh, kh, vv, P, dS, preQ, preK, preV inside the scratch; out[8]: attn_bwd_scratch_floats
extern "C" int probe_attn_bwd_layout(int32_t b, int32_t H, int32_t n, int32_t m, int32_t nnull, int32_t dh,
                                     int64_t* out) {
  float* const base = reinterpret_cast<float*>(alignof(float) * 64);  // any non-null base: only differences are read
  const phk::AttnBwdBufs B = phk::attn_bwd_bufs(base, phk::AttnBwdGeom{b, H, n, m, nnull, dh});
  const float* const p[8] = {B.qh, B.kh, B.vv, B.P, B.dS, B.preQ, B.preK, B.preV};
  for (int i = 0; i < 8; ++i) out[i] = p[i] - base;
  out[8] = phk::attn_bwd_scratch_floats(b, H, n, nnull + m, dh);
  return 0;
}

extern "C" int probe_colsum(const float* x, int64_t rows, int32_t cols, int64_t ld, float* out, phk_stream_t s) {
  return phk::colsum(x, rows, cols, ld, out, phk::to_stream(s));
}
