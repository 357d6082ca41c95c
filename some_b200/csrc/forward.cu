// some_forward: the whole two-head conformer trunk (Gmidi_conform.forward, Gconform.py:119-140, plus the head
// activation of midi_conforms.forward, Gmidi_conform.py:30-40) as ONE C call that enqueues the kernel sequence on the
// caller's stream.  Doing the sequencing natively takes the per-launch host cost from ~50 us of Python + ctypes to a few
// microseconds, which matters for small batches (one 10 s clip is ~50 launches of ~5-20 us each) and lets infer() cut
// big batches into more pipeline chunks.
//
// Per conform_blocke (Gconform.py:56-63), both streams (0 = midi / att1, 1 = bound / att2) in every launch.
//
// ln_fold = 0 (stand-alone LayerNorm launches, 15 per block):
//   LN1 -> GEMM(ffn1.ln1)+SiLU -> GEMM(ffn1.ln2)*0.5+x -> LN2 -> GEMM(to_q|to_kv) -> attention -> GEMM(to_out)+x ->
//   LN3 -> GEMM(pointwise_conv1)+GLU -> dwconv+BN+SiLU -> GEMM(pointwise_conv2)+x -> LN4 -> GEMM(ffn2.ln1)+SiLU ->
//   GEMM(ffn2.ln2)*0.5+x -> LN5
//
// ln_fold = 1 (norm1..norm4 folded into the GEMMs on both sides, 11 per block): every GEMM that writes the residual
// stream in front of a LayerNorm is a PRODUCER (it also writes bf16(x) -> xb and per-row partial sums -> ln_stats), every
// GEMM behind one is a CONSUMER (A = xb, W' = W * gamma, epilogue rstd * (acc - mean * s) + b'):
//   GEMM(ffn1.ln1')+SiLU -> GEMM(ffn1.ln2)*0.5+x [P] -> GEMM(to_q|to_kv') -> attention -> GEMM(to_out)+x [P] ->
//   GEMM(pointwise_conv1')+GLU -> dwconv+BN+SiLU -> GEMM(pointwise_conv2)+x [P] -> GEMM(ffn2.ln1')+SiLU ->
//   GEMM(ffn2.ln2)*0.5+x -> LN5
// norm5 stays a kernel (its output IS the next residual stream).  The stream entering block 0 comes from the input
// projection, so one some_row_stats launch plays the producer there; the Gcf mix GEMM (glu1 / glu2) is the producer in
// front of every later block's norm1.
#include "host_common.h"

#include <vector>

#include "../../include/some_b200.h"

struct some_profiler {
  int capacity = 0;
  int count = 0;
  std::vector<cudaEvent_t> ev;              // 2 per record
  std::vector<some_profile_record> rec;
};

namespace {

constexpr int D = SOME_DIM;
constexpr int FFN = 4 * SOME_DIM;

struct Seq {
  const some_model* m;
  const some_workspace* ws;
  int M, B, max_frames;
  const int32_t* cu;
  some_profiler* prof;
  some_calibration* calib;
  cudaStream_t st;
  int rc = 0;

  // ---- optional per-launch events
  int begin(int kernel, int epi, int n, int k, double work) {
    if (prof == nullptr || prof->count >= prof->capacity) return -1;
    const int i = prof->count++;
    prof->rec[i] = some_profile_record{kernel, epi, n, k, 0.f, work};
    cudaEventRecord(prof->ev[2 * i], st);
    return i;
  }
  void end(int i) {
    if (i >= 0) cudaEventRecord(prof->ev[2 * i + 1], st);
  }

  // calibration pass: column means of the operand the (rounded) weights of this GEMM multiply
  void calibrate(const some_gemm_args& g) {
    if (calib == nullptr || rc) return;
    if (calib->count >= SOME_CALIB_MAX || g.K > SOME_CALIB_K) {
      some::set_error("some_forward: calibration capacity exceeded");
      rc = -1;
      return;
    }
    const int i = calib->count++;
    const bool ln = g.epilogue == SOME_EPI_LN_STORE_BF16 || g.epilogue == SOME_EPI_LN_SILU_BF16 || g.epilogue == SOME_EPI_LN_GLU_BF16;
    calib->k[i] = g.K;
    for (int s = 0; s < 2 && !rc; ++s) {
      const int src = s < g.groups ? s : 0;
      calib->w[i][s] = g.W[src];
      if (s < g.groups)
        rc = some_col_means(g.A[s], M, g.K, g.lda, ln ? g.ln_stats[s] : nullptr, g.ln_parts,
                            calib->means + (static_cast<size_t>(i) * 2 + s) * SOME_CALIB_K, st);
    }
  }

  void gemm(const some_gemm_args& g) {
    calibrate(g);
    if (rc) return;
    const int i = begin(SOME_K_GEMM, g.epilogue, g.N, g.K, 2.0 * M * g.N * g.K * g.groups);
    rc = some_gemm(&g, st);
    end(i);
  }
  some_gemm_args args(const uint16_t* a0, const uint16_t* a1, const uint16_t* w0, const uint16_t* w1, const float* b0,
                      const float* b1, void* o0, void* o1, int n, int k, int ld_out, int epi) const {
    some_gemm_args g{};
    g.A[0] = a0, g.A[1] = a1, g.W[0] = w0, g.W[1] = w1, g.bias[0] = b0, g.bias[1] = b1, g.out[0] = o0, g.out[1] = o1;
    g.groups = 2, g.M = M, g.N = n, g.K = k, g.lda = k, g.ld_out = ld_out, g.epilogue = epi, g.alpha = 1.0f;
    return g;
  }
  // x += alpha * (A . W^T + b)   (in place on the fp32 residual streams); producer = also emit xb / ln_stats
  void resid_gemm(const uint16_t* a0, const uint16_t* a1, const uint16_t* w0, const uint16_t* w1, const float* b0,
                  const float* b1, int n, int k, bool glu, bool producer, float alpha = 1.0f) {
    const int epi = glu ? (producer ? SOME_EPI_GLU_RESID_F32_LN : SOME_EPI_GLU_RESID_F32)
                        : (producer ? SOME_EPI_RESID_F32_LN : SOME_EPI_RESID_F32);
    some_gemm_args g = args(a0, a1, w0, w1, b0, b1, ws->x[0], ws->x[1], n, k, D, epi);
    g.resid[0] = ws->x[0], g.resid[1] = ws->x[1], g.alpha = alpha;
    if (producer) {
      g.out_bf16[0] = ws->xb[0], g.out_bf16[1] = ws->xb[1];
      g.ln_stats[0] = ws->ln_stats[0], g.ln_stats[1] = ws->ln_stats[1];
    }
    gemm(g);
  }
  // LayerNorm-folded consumer: out = epi(LN(x) . W^T + b) computed from xb / ln_stats
  void ln_gemm(const uint16_t* w0, const uint16_t* w1, const float* s0, const float* s1, const float* b0, const float* b1,
               void* o0, void* o1, int n, int ld_out, int epi, int parts) {
    some_gemm_args g = args(ws->xb[0], ws->xb[1], w0, w1, b0, b1, o0, o1, n, D, ld_out, epi);
    g.ln_s[0] = s0, g.ln_s[1] = s1, g.ln_stats[0] = ws->ln_stats[0], g.ln_stats[1] = ws->ln_stats[1], g.ln_parts = parts;
    gemm(g);
  }
  void ln(const some_block_weights& w0, const some_block_weights& w1, int i, bool f32_out) {
    if (rc) return;
    some_ln_args a{};
    a.x[0] = ws->x[0], a.x[1] = ws->x[1];
    a.gamma[0] = w0.ln_g[i], a.gamma[1] = w1.ln_g[i], a.beta[0] = w0.ln_b[i], a.beta[1] = w1.ln_b[i];
    a.out_bf16[0] = ws->a[0], a.out_bf16[1] = ws->a[1];
    if (f32_out) a.out_f32[0] = ws->x[0], a.out_f32[1] = ws->x[1];
    a.groups = 2, a.M = M;
    const int r = begin(SOME_K_LAYERNORM, 0, 0, 0, 2.0 * M * D * (4 + 2 + (f32_out ? 4 : 0)));
    rc = some_layernorm(&a, st);
    end(r);
  }
  void attention() {
    if (rc) return;
    some_attn_args at{};
    at.qkv[0] = ws->qkv[0], at.qkv[1] = ws->qkv[1], at.out[0] = ws->a[0], at.out[1] = ws->a[1];
    at.groups = 2, at.B = B, at.M = M, at.cu_frames = cu, at.max_frames = max_frames;
    const int r = begin(SOME_K_ATTENTION, 0, 0, 0, 0.0);
    rc = some_attention_varlen(&at, st);
    end(r);
  }
  void dwconv(const some_block_weights& w0, const some_block_weights& w1) {
    if (rc) return;
    some_dwconv_args dw{};
    dw.x[0] = ws->g[0], dw.x[1] = ws->g[1], dw.w[0] = w0.w_dw, dw.w[1] = w1.w_dw, dw.b[0] = w0.b_dw, dw.b[1] = w1.b_dw;
    dw.out[0] = ws->a[0], dw.out[1] = ws->a[1];
    dw.groups = 2, dw.B = B, dw.cu_frames = cu, dw.max_frames = max_frames;
    const int r = begin(SOME_K_DWCONV, 0, 0, 0, 2.0 * M * D * 4);                        // bf16 in + bf16 out
    rc = some_dwconv_bn_silu(&dw, st);                                                   // base_conv.py:66-68
    end(r);
  }

  // parts = partial-sum slots of ln_stats describing the stream entering the block (ln_fold only)
  void block(const some_block_weights& w0, const some_block_weights& w1, bool last, int parts) {
    const bool fold = m->ln_fold != 0;
    for (int f = 0; f < 2; ++f) {
      if (f == 1) {
        // ---- attention module (Gconform.py:58) and conv module (:59-61) between the two half-step FFNs
        if (fold) {
          ln_gemm(w0.w_qkvf, w1.w_qkvf, w0.s_qkv, w1.s_qkv, w0.b_qkvf, w1.b_qkvf, ws->qkv[0], ws->qkv[1], 3 * D, 3 * D,
                  SOME_EPI_LN_STORE_BF16, parts);
        } else {
          ln(w0, w1, 1, false);
          gemm(args(ws->a[0], ws->a[1], w0.w_qkv, w1.w_qkv, nullptr, nullptr, ws->qkv[0], ws->qkv[1], 3 * D, D, 3 * D,
                    SOME_EPI_STORE_BF16));
        }
        attention();
        resid_gemm(ws->a[0], ws->a[1], w0.w_out, w1.w_out, w0.b_out, w1.b_out, D, D, false, fold);      // :60
        if (fold) {
          ln_gemm(w0.w_pw1f, w1.w_pw1f, w0.s_pw1, w1.s_pw1, w0.b_pw1f, w1.b_pw1f, ws->g[0], ws->g[1], 2 * D, D,
                  SOME_EPI_LN_GLU_BF16, 4);
        } else {
          ln(w0, w1, 2, false);
          gemm(args(ws->a[0], ws->a[1], w0.w_pw1, w1.w_pw1, w0.b_pw1, w1.b_pw1, ws->g[0], ws->g[1], 2 * D, D, D,
                    SOME_EPI_GLU_BF16));                                                                // base_conv.py:65
        }
        dwconv(w0, w1);
        resid_gemm(ws->a[0], ws->a[1], w0.w_pw2, w1.w_pw2, w0.b_pw2, w1.b_pw2, D, D, false, fold);      // base_conv.py:69 + :61
        parts = 4;
      }
      // ---- ffn1 (:57) / ffn2 (:62): x += 0.5 * ln2(SiLU(ln1(norm(x))))
      if (fold) {
        ln_gemm(w0.ffn_w1f[f], w1.ffn_w1f[f], w0.ffn_s1[f], w1.ffn_s1[f], w0.ffn_b1f[f], w1.ffn_b1f[f], ws->h[0], ws->h[1],
                FFN, FFN, SOME_EPI_LN_SILU_BF16, parts);
      } else {
        ln(w0, w1, f == 0 ? 0 : 3, false);
        gemm(args(ws->a[0], ws->a[1], w0.ffn_w1[f], w1.ffn_w1[f], w0.ffn_b1[f], w1.ffn_b1[f], ws->h[0], ws->h[1], FFN, D,
                  FFN, SOME_EPI_SILU_BF16));
      }
      // ffn1's output feeds norm2 (producer); ffn2's feeds norm5, which stays a kernel
      resid_gemm(ws->h[0], ws->h[1], w0.ffn_w2[f], w1.ffn_w2[f], w0.ffn_b2[f], w1.ffn_b2[f], D, FFN, false, fold && f == 0,
                 0.5f);
      parts = 4;
    }
    if (!last) {
      ln(w0, w1, 4, true);                                                               // :63, residual of the next Gcf
    } else if (!rc) {
      // final pair: midi stream -> normalised bf16 for outln; bound stream -> fused norm5 + cutheard + sigmoid
      some_ln_args a{};
      a.x[0] = a.x[1] = ws->x[0], a.gamma[0] = a.gamma[1] = w0.ln_g[4], a.beta[0] = a.beta[1] = w0.ln_b[4];
      a.out_bf16[0] = a.out_bf16[1] = ws->a[0];
      a.groups = 1, a.M = M;
      int r = begin(SOME_K_LAYERNORM, 0, 0, 0, 1.0 * M * D * 6);
      rc = some_layernorm(&a, st);
      end(r);
      if (!rc) {
        r = begin(SOME_K_BOUND_HEAD, 0, 0, 0, 1.0 * M * D * 4);
        rc = some_bound_head(ws->x[1], w1.ln_g[4], w1.ln_b[4], m->w_cut, m->b_cut, M, ws->bounds, st);
        end(r);
      }
    }
  }
};

}  // namespace

extern "C" int some_forward(const some_model* m, const some_workspace* ws, int M, int B, const int32_t* cu_frames,
                            int max_frames, int head, some_profiler* prof, some_calibration* calib, cudaStream_t stream) {
  SOME_REQUIRE(m != nullptr && ws != nullptr && cu_frames != nullptr, "some_forward: null argument");
  SOME_REQUIRE(m->blocks != nullptr && m->lay >= 0 && m->outdim >= 1 && m->outdim <= 256, "some_forward: bad model");
  SOME_REQUIRE(head == SOME_EPI_SIGMOID_F32 || head == SOME_EPI_SOFTMAX_F32 || head == SOME_EPI_BIAS_F32,
               "some_forward: head must be SOME_EPI_SIGMOID_F32 / SOME_EPI_SOFTMAX_F32 / SOME_EPI_BIAS_F32 (got %d)", head);
  const bool fold = m->ln_fold != 0;
  if (fold)
    SOME_REQUIRE(ws->xb[0] && ws->xb[1] && ws->ln_stats[0] && ws->ln_stats[1],
                 "some_forward: ln_fold needs some_workspace.xb and ln_stats");
  if (M <= 0 || B <= 0) return 0;
  if (calib != nullptr) {
    SOME_REQUIRE(calib->means != nullptr, "some_forward: calibration without a means buffer");
    calib->count = 0;
  }
  Seq s{m, ws, M, B, max_frames, cu_frames, prof, calib, stream};
  // inln / inln1 (Gconform.py:122-125): both streams read the same units
  {
    some_gemm_args g = s.args(ws->units, ws->units, m->w_in[0], m->w_in[1], m->b_in[0], m->b_in[1], ws->x[0], ws->x[1], D,
                              SOME_N_MELS, D, SOME_EPI_BIAS_F32);
    s.gemm(g);
  }
  int parts = 0;
  if (fold && !s.rc) {
    some_rowstats_args a{};
    a.x[0] = ws->x[0], a.x[1] = ws->x[1], a.out_bf16[0] = ws->xb[0], a.out_bf16[1] = ws->xb[1];
    a.ln_stats[0] = ws->ln_stats[0], a.ln_stats[1] = ws->ln_stats[1], a.groups = 2, a.M = M;
    const int r = s.begin(SOME_K_ROW_STATS, 0, 0, 0, 2.0 * M * D * 6);
    s.rc = some_row_stats(&a, stream);
    s.end(r);
    parts = 1;
  }
  for (int i = 0; i < m->lay; ++i) {
    s.block(m->blocks[2 * i], m->blocks[2 * i + 1], false, parts);
    // Gcf.forward :85-87: midi += GLU(glu2(bound)); bound += GLU(glu1(midi))   (ws->a = bf16 copies of the norm5 outputs)
    s.resid_gemm(ws->a[1], ws->a[0], m->glu_w[2 * i + 1], m->glu_w[2 * i], m->glu_b[2 * i + 1], m->glu_b[2 * i], 2 * D, D,
                 true, fold);
    parts = SOME_LN_SLOTS;
  }
  s.block(m->blocks[2 * m->lay], m->blocks[2 * m->lay + 1], true, parts);
  {
    some_gemm_args g = s.args(ws->a[0], ws->a[0], m->w_head, m->w_head, m->b_head, m->b_head, ws->probs, ws->probs,
                              m->outdim, D, m->outdim, head);                            // outln (+ sigmoid / softmax)
    g.groups = 1;
    s.calibrate(g);
    if (!s.rc) {
      const int i = s.begin(SOME_K_GEMM, head, m->outdim, D, 2.0 * M * m->outdim * D);
      s.rc = some_gemm(&g, stream);
      s.end(i);
    }
  }
  return s.rc;
}

// ---------------------------------------------------------------------------------------------------- profiler
extern "C" int some_profiler_create(int capacity, some_profiler** out) {
  SOME_REQUIRE(out != nullptr && capacity > 0 && capacity <= (1 << 20), "some_profiler_create: bad arguments");
  some_profiler* p = new some_profiler();
  p->capacity = capacity;
  p->ev.resize(2 * static_cast<size_t>(capacity));
  p->rec.resize(capacity);
  for (auto& e : p->ev) {
    if (cudaEventCreate(&e) != cudaSuccess) {
      some::set_error("some_profiler_create: cudaEventCreate failed");
      return -2;   // (events created so far leak; this only happens when the context is already broken)
    }
  }
  *out = p;
  return 0;
}
extern "C" int some_profiler_destroy(some_profiler* p) {
  if (p == nullptr) return 0;
  for (auto& e : p->ev) cudaEventDestroy(e);
  delete p;
  return 0;
}
extern "C" int some_profiler_reset(some_profiler* p) {
  SOME_REQUIRE(p != nullptr, "some_profiler_reset: null profiler");
  p->count = 0;
  return 0;
}
extern "C" int some_profiler_read(some_profiler* p, int cap, some_profile_record* out) {
  SOME_REQUIRE(p != nullptr && (out != nullptr || cap == 0), "some_profiler_read: bad arguments");
  for (int i = 0; i < p->count && i < cap; ++i) {
    cudaError_t e = cudaEventSynchronize(p->ev[2 * i + 1]);
    SOME_REQUIRE(e == cudaSuccess, "some_profiler_read: %s", cudaGetErrorString(e));
    float ms = 0.f;
    e = cudaEventElapsedTime(&ms, p->ev[2 * i], p->ev[2 * i + 1]);
    SOME_REQUIRE(e == cudaSuccess, "some_profiler_read: %s", cudaGetErrorString(e));
    out[i] = p->rec[i];
    out[i].ms = ms;
  }
  return p->count;
}

// ---------------------------------------------------------------------------------------------------- workspace sizing
namespace {
uint64_t carve(some::Carver& c, int M, int outdim, int ln_fold, some_workspace* ws) {
  const uint64_t m = static_cast<uint64_t>(M > 0 ? M : 0);
  some_workspace w{};
  for (int s = 0; s < 2; ++s) w.x[s] = c.take<float>(m * D * 4);
  for (int s = 0; s < 2; ++s) w.a[s] = c.take<uint16_t>(m * D * 2);
  for (int s = 0; s < 2; ++s) w.h[s] = c.take<uint16_t>(m * FFN * 2);
  for (int s = 0; s < 2; ++s) w.qkv[s] = c.take<uint16_t>(m * 3 * D * 2);
  for (int s = 0; s < 2; ++s) w.g[s] = c.take<uint16_t>(m * D * 2);
  w.units = c.take<uint16_t>(m * SOME_N_MELS * 2);
  w.probs = c.take<float>(m * static_cast<uint64_t>(outdim) * 4);
  w.bounds = c.take<float>(m * 4);
  if (ln_fold) {
    for (int s = 0; s < 2; ++s) w.xb[s] = c.take<uint16_t>(m * D * 2);
    for (int s = 0; s < 2; ++s) w.ln_stats[s] = c.take<float>(m * SOME_LN_SLOTS * 2 * 4);
  }
  if (ws != nullptr) *ws = w;
  return c.off;
}
}  // namespace

extern "C" uint64_t some_workspace_bytes(int M, int outdim, int ln_fold) {
  some::Carver c{nullptr};
  return carve(c, M, outdim, ln_fold, nullptr);
}
extern "C" int some_workspace_carve(void* device_block, uint64_t bytes, int M, int outdim, int ln_fold, some_workspace* ws) {
  SOME_REQUIRE(device_block != nullptr && ws != nullptr && M > 0 && outdim >= 1 && outdim <= 256, "some_workspace_carve: bad arguments");
  SOME_REQUIRE((reinterpret_cast<uintptr_t>(device_block) & 255) == 0, "some_workspace_carve: the block must be 256-byte aligned");
  SOME_REQUIRE(bytes >= some_workspace_bytes(M, outdim, ln_fold), "some_workspace_carve: block of %llu bytes is too small for M=%d",
               (unsigned long long)bytes, M);
  some::Carver c{static_cast<uint8_t*>(device_block)};
  carve(c, M, outdim, ln_fold, ws);
  return 0;
}
