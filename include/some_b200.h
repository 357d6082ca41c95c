/* some_b200.h — C ABI of libsome_b200.so: the H100 (sm_90a) kernels behind SOME's inference hot path.
 *
 * The reference (openvpi/SOME) is pure Python/PyTorch and has NO native FFI; the
 * "operator interface" of this path is the set of torch calls listed below.  Each entry point names
 * the reference call site (file:line in the reference repository) it replaces.  INTEGRATION.md shows the
 * ctypes binding the reference's inference/ package uses to call them.
 *
 * Conventions
 *   - every function returns 0 on success, < 0 on error; some_last_error() returns a thread-local message;
 *   - all buffers are CALLER-allocated device memory (torch tensors -> data_ptr()); the library never
 *     allocates, frees or retains them; no torch / ATen types cross this boundary;
 *   - all work is enqueued on the caller's stream; no hidden synchronisation;
 *   - "bf16" buffers are raw uint16 bfloat16; row-major; M = total frames of a packed (var-len) batch;
 *   - cu_frames[B + 1] (int32, device) = prefix sums of per-clip frame counts (clip b = rows
 *     [cu_frames[b], cu_frames[b + 1])).  Clips never interact: attention, depthwise conv and decode are
 *     per clip, exactly like the reference's batch-1 loop (inference/base_infer.py:46-53).
 */
#ifndef SOME_B200_H_
#define SOME_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SOME_B200_VERSION 202

#ifndef __CUDA_RUNTIME_H__
typedef struct CUstream_st* cudaStream_t;
#endif

/* Model geometry the kernels are specialised for (all shipped configs: configs/*.yaml). */
#define SOME_DIM 512
#define SOME_HEADS 8
#define SOME_HEAD_DIM 64
#define SOME_CONV_K 31
#define SOME_N_MELS 80
#define SOME_N_FFT 2048
#define SOME_HOP 512
#define SOME_MEL_BINS 372 /* spectrum bins 0..371 carry all non-zero mel weights (fmax = 8 kHz) */
#define SOME_MEL_MAXW 24  /* widest mel filter, in bins */
#define SOME_MEL_TW 1396  /* complex twiddles: W_1024^(n2 k1) at [k1 * 32 + n2] (1024), then W_2048^k for k < 372 */

int some_version(void);
const char* some_last_error(void);
/* Programmatic dependent launch for the CALLING thread's subsequent launches of the trunk kernels (some_gemm, some_layernorm,
 * some_attention_varlen, some_dwconv_bn_silu, some_bound_head, and through them some_forward): a kernel may become resident and
 * run its prologue while its predecessor in the stream is still running; it touches activations only after the predecessor has
 * completed (griddepcontrol.wait).  Pays on small batches (a step is ~70 dependent launches of a few microseconds each); works
 * under stream capture.  Returns the previous setting.  No reference counterpart. */
int some_set_pdl(int on);

/* ---- K-mel: modules/rmvpe/spec.py:38-72 (F.pad 1024/1024, torch.stft n_fft 2048 hop 512 periodic Hann,
 * abs, mel_basis matmul, log(clamp 1e-5)) + the transpose at inference/me_infer.py:31.
 *   wave          f32, all clips in one buffer (clip starts may be padded for 16-byte alignment)
 *   clip_start    int64 [B], first sample of each clip in `wave`;  clip_len int64 [B], samples L_b
 *   cu_frames     int32 [B + 1], T_b = 1 + L_b / 512
 *   max_frames    max_b T_b (grid sizing: ceil(max_frames / 32) CTAs per clip)
 *   mel_start     int32 [80]: first spectrum bin with non-zero weight in filter m
 *   mel_count     int32 [80]: number of contiguous non-zero bins (<= SOME_MEL_MAXW)
 *   mel_weights   f32 [80][SOME_MEL_MAXW]: those weights (librosa htk / slaney filterbank, spec.py:22-28)
 *   twiddle       f32 [SOME_MEL_TW][2] (cos, sin), host-computed in double: exp(-2 pi i n2 k1 / 1024) at [k1 * 32 + n2]
 *                 (between the two 32-point passes of the 32 x 32 FFT), then exp(-2 pi i k / 2048) for k < 372 (real-FFT
 *                 unpack)
 *   window        f32 [2048] periodic Hann (torch.hann_window)
 *   out_f32       f32 [M, 80] or NULL;  out_bf16  bf16 [M, 80] or NULL (A operand of the input projections) */
int some_mel_logmel(const float* wave, const int64_t* clip_start, const int64_t* clip_len,
                    const int32_t* cu_frames, int B, int max_frames,
                    const int32_t* mel_start, const int32_t* mel_count, const float* mel_weights,
                    const float* twiddle, const float* window, float* out_f32, uint16_t* out_bf16, float clamp,
                    cudaStream_t stream);

/* ---- K-mel-keyshift (SURVEY.md §8f-4): MelSpectrogram.forward with keyshift != 0 and / or speed != 1
 * (modules/rmvpe/spec.py:38-72; caller preprocessing/me_binarizer.py:235-247): n_fft = win_length = round(2048 * 2^(keyshift /
 * 12)), hop = round(512 * speed), F.pad(pad_left = win / 2 (0 when center=False), ...), periodic Hann of n_fft points,
 * magnitudes of bins 0..371 scaled by mag_scale = 2048 / n_fft (spec.py:68), same filterbank and log(clamp).
 *   cu_frames  int32 [B + 1], T_b = 1 + (L_b + pad_left + pad_right - n_fft) / hop (= 1 + L_b / hop when center=True)
 *   twiddle    f32 [n_fft][2] = exp(-2 pi i m / n_fft), host-computed in double;  window f32 [n_fft] */
int some_mel_logmel_keyshift(const float* wave, const int64_t* clip_start, const int64_t* clip_len,
                             const int32_t* cu_frames, int B, int max_frames, int n_fft, int hop, int pad_left,
                             float mag_scale, const int32_t* mel_start, const int32_t* mel_count,
                             const float* mel_weights, const float* twiddle, const float* window, float* out_f32,
                             uint16_t* out_bf16, float clamp, cudaStream_t stream);

/* ---- K-ln: nn.LayerNorm(512), eps 1e-5 (Gconform.py:57-63 norm1..norm5) over rows of x f32 [M, 512].
 *   out_bf16: normalised rows as bf16 (A operand of the next GEMM) or NULL
 *   out_f32 : normalised rows as f32 (the residual stream after norm5) or NULL (may alias x)
 * groups = 1 or 2 independent problems (midi / bound stream) in one launch. */
typedef struct {
  const float* x[2];
  const float* gamma[2];
  const float* beta[2];
  uint16_t* out_bf16[2];
  float* out_f32[2];
  int groups;
  int M;
} some_ln_args;
int some_layernorm(const some_ln_args* args, cudaStream_t stream);

/* ---- K-gemm: C = epilogue(A[M,K] . W[N,K]^T), bf16 operands, fp32 accumulation on the tensor cores (wgmma).
 * Replaces every nn.Linear / 1x1 Conv1d of the trunk (see gemm.cu header for the call sites). */
enum some_epilogue {
  SOME_EPI_STORE_BF16 = 0,     /* out bf16 [M,N]   = acc (+ bias)                       to_q|to_kv          */
  SOME_EPI_SILU_BF16 = 1,      /* out bf16 [M,N]   = silu(acc + bias)                   ffn.ln1 + act       */
  SOME_EPI_GLU_BF16 = 2,       /* out bf16 [M,N/2] = (a + b_a) * sigmoid(g + b_g)       pointwise_conv1+GLU */
  SOME_EPI_RESID_F32 = 3,      /* out f32 [M,N]    = alpha * (acc + bias) + resid       ffn.ln2/to_out/pw2  */
  SOME_EPI_GLU_RESID_F32 = 4,  /* out f32 [M,N/2]  = resid + glu(acc + bias)            Gcf glu1/glu2       */
  SOME_EPI_BIAS_F32 = 5,       /* out f32 [M,N]    = acc + bias                         inln/inln1, logits  */
  SOME_EPI_SIGMOID_F32 = 6,    /* out f32 [M,N]    = sigmoid(acc + bias)                outln + sig         */
  SOME_EPI_SOFTMAX_F32 = 7,    /* out f32 [M,N]    = softmax_row(acc + bias), N <= 256  outln + softmax     */
  /* LayerNorm folded into the GEMMs around it (norm1..norm4 of conform_blocke, Gconform.py:57-62).
   * Producers: the residual GEMM in front of the LayerNorm also writes bf16(out) and, per row, partial (sum x, sum x^2)
   * over each 128-column slice of its output.  Consumers: A = bf16(x) (NOT normalised), W' = W * gamma (per column k),
   * ln_s[n] = sum_k W'[n,k], bias' = bias + W . beta; the epilogue applies  rstd * (acc - mean * ln_s[n]) + bias'[n]
   * (= LayerNorm(x) . W^T + bias up to rounding) before the activation. */
  SOME_EPI_LN_STORE_BF16 = 8,      /* consumer of SOME_EPI_STORE_BF16        to_q|to_kv after norm2        */
  SOME_EPI_LN_SILU_BF16 = 9,       /* consumer of SOME_EPI_SILU_BF16         ffn.ln1 after norm1 / norm4   */
  SOME_EPI_LN_GLU_BF16 = 10,       /* consumer of SOME_EPI_GLU_BF16          pointwise_conv1 after norm3   */
  SOME_EPI_RESID_F32_LN = 11,      /* producer variant of SOME_EPI_RESID_F32                               */
  SOME_EPI_GLU_RESID_F32_LN = 12   /* producer variant of SOME_EPI_GLU_RESID_F32                           */
};
#define SOME_LN_SLOTS 8 /* partial-sum slots per row in ln_stats: f32 [M][SOME_LN_SLOTS][2] */
/* GLU epilogues expect W rows (and bias) packed in 32-row groups: 16 "out" rows followed by their 16
 * "gate" rows (host packing: some_b200/weights.py).  bias arrays are padded to a multiple of 32 floats. */
typedef struct {
  const uint16_t* A[2]; /* bf16 [M, K], row pitch lda */
  const uint16_t* W[2]; /* bf16 [N, K] */
  const float* bias[2]; /* f32 [N] or NULL */
  void* out[2];
  const float* resid[2];
  int groups, M, N, K, lda, ld_out, epilogue;
  float alpha;
  /* LayerNorm folding (SOME_EPI_LN_* / SOME_EPI_*_LN only; ignored otherwise) */
  const float* ln_s[2];  /* consumers: f32 [N] column sums of W' (packed like bias) */
  float* ln_stats[2];    /* producers write, consumers read: f32 [M][SOME_LN_SLOTS][2] partial (sum x, sum x^2) */
  int ln_parts;          /* consumers: valid slots per row (4 after a RESID producer, 8 after a GLU_RESID one, 1 after
                            some_row_stats) */
  uint16_t* out_bf16[2]; /* producers: bf16 [M, ld_out] copy of out (the consumers' A operand) */
} some_gemm_args;
int some_gemm(const some_gemm_args* args, cudaStream_t stream);

/* ---- K-rowstats: LayerNorm-producer side for a residual stream no producer GEMM has written (the input projection in
 * front of block 0, Gconform.py:124-125 -> norm1 at :57): out_bf16 = bf16(x), ln_stats[row][0] = (sum x, sum x^2);
 * the consumer GEMM then runs with ln_parts = 1. */
typedef struct {
  const float* x[2];      /* f32 [M, 512] */
  uint16_t* out_bf16[2];  /* bf16 [M, 512] */
  float* ln_stats[2];     /* f32 [M][SOME_LN_SLOTS][2] */
  int groups, M;
} some_rowstats_args;
int some_row_stats(const some_rowstats_args* args, cudaStream_t stream);

/* ---- K-attn: F.scaled_dot_product_attention(q, k, v), no mask, scale 64^-0.5, per clip
 * (base_attention.py:34-45 incl. both rearranges).  qkv bf16 [M, 1536] = [q(8x64) | k(8x64) | v(8x64)]
 * as written by the fused to_q|to_kv GEMM; out bf16 [M, 512] = 'b h t c -> b t (h c)'. */
typedef struct {
  const uint16_t* qkv[2];
  uint16_t* out[2];
  int groups;
  int B, M;                 /* clips, total rows of qkv (rows >= M are never read: TMA zero-fills them) */
  const int32_t* cu_frames; /* device int32 [B + 1] */
  int max_frames;           /* max_b T_b: grid = ceil(max_frames / 128) query tiles per clip */
} some_attn_args;
int some_attention_varlen(const some_attn_args* args, cudaStream_t stream);

/* ---- K-dwconv: depthwise Conv1d(k=31, pad 15, groups=512) + BatchNorm1d(eval) + SiLU
 * (base_conv.py:66-68) on the packed [M, 512] bf16 layout (no transposes), zero halo per clip.
 *   w  f32 [31][512] taps with the BN scale folded in;  b f32 [512] = folded bias */
typedef struct {
  const uint16_t* x[2];
  const float* w[2];
  const float* b[2];
  uint16_t* out[2]; /* must not alias x (neighbouring tiles read the halo) */
  int groups;
  int B;
  const int32_t* cu_frames; /* device int32 [B + 1] */
  int max_frames;           /* max_b T_b: grid = ceil(max_frames / 128) tiles per clip (tiles never span clips) */
} some_dwconv_args;
int some_dwconv_bn_silu(const some_dwconv_args* args, cudaStream_t stream);

/* ---- K-boundhead: norm5 of the bound stream's last block + cutheard Linear(512,1) + sigmoid
 * (Gconform.py:63,135,137-138).  x f32 [M,512] -> bounds f32 [M]. */
int some_bound_head(const float* x, const float* gamma, const float* beta, const float* w, float bias, int M,
                    float* bounds, cudaStream_t stream);

/* ---- K-decode: utils/infer_utils.py:9-76 + inference/me_infer.py:78-97 (continuous) and
 * inference/me_quant_infer.py:21-38 (quantized: argmax over 129 bins, rest = bin 128); three launches: frames (grid over all M rows), per-clip
 * alignment, per-note reduction.  cu_frames must cover rows [0, M).
 *   probs f32 [M, N] (N = 128 sigmoid bins / 129 softmax bins), bounds f32 [M]
 *   outputs are packed per clip at offset cu_frames[b] (a clip never has more notes than frames):
 *     note_midi f32 [M], note_dur i32 [M] (frames; seconds = dur * hop / sr on the host, me_infer.py:95),
 *     note_rest u8 [M], note_count i32 [B]
 *   optional debug outputs (may be NULL): frame2item i32 [M], values f32 [M], rest u8 [M]
 * Integer outputs match the CPU reference exactly for identical inputs: the boundary cumsum is accumulated
 * sequentially in double and rounded per prefix like ATen's CPU cumsum; per-note sums run in frame order. */
typedef struct {
  const float* probs;
  const float* bounds;
  const int32_t* cu_frames;
  int B, M, N;
  int quantized;
  float vmin, vmax, deviation, threshold; /* midi_min, midi_max, midi_prob_deviation, rest_threshold */
  float* note_midi;
  int32_t* note_dur;
  uint8_t* note_rest;
  int32_t* note_count;
  int32_t* dbg_frame2item;
  float* dbg_values;
  uint8_t* dbg_rest;
  void* scratch; /* device, >= some_decode_scratch_bytes(M) */
} some_decode_args;
uint64_t some_decode_scratch_bytes(int M);
int some_decode_notes(const some_decode_args* args, cudaStream_t stream);

/* ---- K-rms (row §8f-1, the step in front of the path): short-time RMS for the silence slicer.
 * Replaces get_rms (utils/slicer2.py:5-38) as called by Slicer.slice (slicer2.py:81): zero padding of frame_length / 2 on
 * both sides, frames of frame_length samples every hop samples, sqrt(mean(x^2)) in float32 with numpy's pairwise summation
 * order, i.e. BIT-identical to the reference so the host state machine (slicer2.py:84-133) cuts identical chunks.
 * wave: device f32 [n_samples] (the whole recording, resident; the chunks are later processed in place);
 * rms: device f32 [n_frames], n_frames = 1 + (n_samples + 2 * (frame_length / 2) - frame_length) / hop. */
int some_slicer_rms(const float* wave, long long n_samples, int frame_length, int hop, float* rms, int n_frames,
                    cudaStream_t stream);

/* ---- some_forward: the whole trunk Gmidi_conform.forward (Gconform.py:119-140) + head activation
 * (Gmidi_conform.py:30-40) as one call that enqueues the launch sequence above on `stream`.
 * All pointers are device pointers owned by the caller (packed by some_b200/weights.py); the structs themselves are
 * host memory and are only read during the call. */
typedef struct {
  const float* ln_g[5];        /* norm1..norm5 weight / bias, f32 [512] */
  const float* ln_b[5];
  const uint16_t* ffn_w1[2];   /* ffn1 / ffn2: ln1 bf16 [2048,512], ln2 bf16 [512,2048] */
  const float* ffn_b1[2];
  const uint16_t* ffn_w2[2];
  const float* ffn_b2[2];
  const uint16_t* w_qkv;       /* bf16 [1536,512] = to_q | to_kv */
  const uint16_t* w_out;       /* bf16 [512,512] */
  const float* b_out;
  const uint16_t* w_pw1;       /* bf16 [1024,512], GLU-packed rows */
  const float* b_pw1;
  const float* w_dw;           /* f32 [31][512], BatchNorm folded */
  const float* b_dw;
  const uint16_t* w_pw2;       /* bf16 [512,512] */
  const float* b_pw2;
  /* LayerNorm-folded consumers (used when some_model.ln_fold != 0; see SOME_EPI_LN_*): W' = bf16(W * gamma_k),
   * s[n] = sum_k W'[n,k], b' = bias + W . beta.  norm1 -> ffn1.ln1, norm4 -> ffn2.ln1, norm2 -> to_q|to_kv,
   * norm3 -> pointwise_conv1 (GLU-packed like w_pw1).  norm5 is never folded (its output is the residual stream). */
  const uint16_t* ffn_w1f[2];
  const float* ffn_s1[2];
  const float* ffn_b1f[2];
  const uint16_t* w_qkvf;
  const float* s_qkv;
  const float* b_qkvf;
  const uint16_t* w_pw1f;
  const float* s_pw1;
  const float* b_pw1f;
} some_block_weights;
typedef struct {
  int lay, outdim;
  const uint16_t* w_in[2];     /* inln / inln1 bf16 [512,80] */
  const float* b_in[2];
  const some_block_weights* blocks; /* host array [(lay + 1) * 2]: entry 2 i + s = block i of stream s (0 = att1, 1 = att2) */
  const uint16_t* const* glu_w;     /* host array [lay * 2]: entry 2 i + 0 = glu1 (fed by midi), 2 i + 1 = glu2, GLU-packed */
  const float* const* glu_b;
  const uint16_t* w_head;      /* outln bf16 [outdim,512] */
  const float* b_head;         /* f32, padded to a multiple of 32 */
  const float* w_cut;          /* cutheard f32 [512] */
  float b_cut;
  int ln_fold;                 /* != 0: norm1..norm4 folded into the GEMMs around them (needs the *f / s_* fields above and
                                  some_workspace.xb / ln_stats); 0: stand-alone LayerNorm launches */
} some_model;
typedef struct {
  float* x[2];                 /* f32 [M,512] residual streams */
  uint16_t* a[2];              /* bf16 [M,512] */
  uint16_t* h[2];              /* bf16 [M,2048] */
  uint16_t* qkv[2];            /* bf16 [M,1536] */
  uint16_t* g[2];              /* bf16 [M,512] */
  const uint16_t* units;       /* bf16 [M,80] log-mel (input) */
  float* probs;                /* f32 [M,outdim] (output) */
  float* bounds;               /* f32 [M] (output) */
  uint16_t* xb[2];             /* bf16 [M,512] copy of the residual stream (ln_fold only) */
  float* ln_stats[2];          /* f32 [M][SOME_LN_SLOTS][2] (ln_fold only) */
} some_workspace;
/* Workspace sizing for hosts that do not use the Python engine: the number of bytes some_workspace needs for M rows (every
 * buffer 256-byte aligned, ln_fold buffers included when ln_fold != 0), and a helper that carves ONE caller-allocated device
 * block of that size into the struct (units / probs / bounds included).  Returns 0 / fills *ws on success. */
uint64_t some_workspace_bytes(int M, int outdim, int ln_fold);
int some_workspace_carve(void* device_block, uint64_t bytes, int M, int outdim, int ln_fold, some_workspace* ws);

/* ---- Checkpoint packing for hosts that do not use some_b200/weights.py: HOST memory in, HOST memory out, no CUDA call.  The
 * caller reads the checkpoint (`torch.load(path)['state_dict']`, `model.` prefix: base_infer.py:27-33), calls these, uploads the
 * results and fills some_model / the table arguments of some_mel_logmel.  (csrc/pack.cu; each mirrors one step of weights.py.)
 *   some_pack_bf16      fp32 -> bf16, round to nearest even (every GEMM weight: nn.Linear's [N][K] layout is the B operand as is)
 *   some_pack_glu_rows  rows [out 0..C-1 | gate C..2C-1] -> groups of 32 rows, 16 out rows then their 16 gates: the row order
 *                       of the GLU producers (pointwise_conv1 base_conv.py:65, glu1 / glu2 Gconform.py:85-87), weights AND biases
 *   some_pack_dwconv_bn depthwise_conv weight [C][K] + bias and BatchNorm1d running statistics (eval, eps 1e-5) ->
 *                       taps [K][C] and bias [C] of some_dwconv_bn_silu (base_conv.py:66-67); float64 inside
 *   some_pack_ln_fold   LayerNorm (gamma, beta) folded into the following Linear for the SOME_EPI_LN_* epilogues:
 *                       w_out = bf16(W gamma) [N][K] (GLU row order if glu_rows), s_out[n] = sum_k w_out[n][k], b_out = W beta + bias
 *   some_mel_tables     librosa.filters.mel(sr, 2048, 80, fmin, fmax, htk=True) with the Slaney normalisation (spec.py:22-28) as the
 *                       sparse tables of some_mel_logmel: mel_start / mel_count [80], mel_weights [80][SOME_MEL_MAXW], the FFT
 *                       twiddles [SOME_MEL_TW][2] and the periodic Hann window [2048] (spec.py:45); fails if a filter does not fit */
int some_pack_bf16(const float* src, long long n, uint16_t* dst);
int some_pack_glu_rows(const void* src, int elem_bytes, int rows, long long row_elems, void* dst);
int some_pack_dwconv_bn(const float* dw_weight, const float* dw_bias, const float* bn_weight, const float* bn_bias,
                        const float* bn_mean, const float* bn_var, int channels, int taps, float* out_taps, float* out_bias);
int some_pack_ln_fold(const float* w, const float* bias, const float* gamma, const float* beta, int n, int k, int glu_rows,
                      uint16_t* w_out, float* s_out, float* b_out);
int some_mel_tables(int sample_rate, int n_fft, int n_mels, double fmin, double fmax, int32_t* mel_start, int32_t* mel_count,
                    float* mel_weights, float* twiddle, float* window);

/* Optional per-launch timing of some_forward (bench.py's roofline pass): CUDA events on the launching stream around every
 * kernel the sequencer enqueues.  The library owns the events; read after the stream has been synchronised. */
typedef struct some_profiler some_profiler;
enum some_kernel_id {
  SOME_K_GEMM = 0, SOME_K_ATTENTION = 1, SOME_K_LAYERNORM = 2, SOME_K_DWCONV = 3, SOME_K_BOUND_HEAD = 4, SOME_K_ROW_STATS = 5
};
typedef struct {
  int kernel;   /* enum some_kernel_id */
  int epilogue; /* GEMM: enum some_epilogue, else 0 */
  int n, k;     /* GEMM shape (M is the call's), else 0 */
  float ms;     /* device time between the two events */
  double work;  /* GEMM: 2 M N K groups FLOP; row-wise kernels: algorithmic bytes; attention: 0 (depends on the clip lengths,
                   which live on the device: the caller knows them) */
} some_profile_record;
int some_profiler_create(int capacity, some_profiler** out);
int some_profiler_destroy(some_profiler* prof);
int some_profiler_reset(some_profiler* prof);
/* Synchronises on the recorded events; fills up to `cap` records in launch order; returns the number recorded (< 0: error). */
int some_profiler_read(some_profiler* prof, int cap, some_profile_record* out);

/* Optional calibration pass (load time, some_b200/weights.py: bias correction for the bf16 rounding of the weights): while the
 * sequencer runs on a calibration batch it also computes, for every GEMM, the column means over the M rows of the operand
 * the rounded weights multiply — A itself, or the normalised rows (x - mean) * rstd for the LayerNorm-folded consumers —
 * so that the host can add  (W - bf16(W)) . E[a]  to the layer's bias: the rounding of W is a FIXED perturbation of the
 * model whose mean effect on the outputs would otherwise accumulate in the decoder's boundary cumsum (utils/infer_utils.py:28). */
#define SOME_CALIB_MAX 512
#define SOME_CALIB_K 2048
typedef struct {
  float* means;   /* device f32 [SOME_CALIB_MAX][2][SOME_CALIB_K] */
  int count;      /* out: GEMMs recorded (launch order) */
  const void* w[SOME_CALIB_MAX][2]; /* out: the W pointers of GEMM i (identify the layer; equal for 1-group launches) */
  int k[SOME_CALIB_MAX];            /* out: its K */
} some_calibration;
/* out[k] = mean over rows of a[row, k] (stats == NULL) or of (a[row, k] - mean_row) * rstd_row (row statistics from
 * ln_stats / parts as in the SOME_EPI_LN_* epilogues).  a bf16 [M, K] with row pitch lda. */
int some_col_means(const uint16_t* a, int M, int K, int lda, const float* ln_stats, int ln_parts, float* out,
                   cudaStream_t stream);

/* head: SOME_EPI_SIGMOID_F32 (sig=True), SOME_EPI_SOFTMAX_F32 (softmax=True) or SOME_EPI_BIAS_F32 (raw logits);
 * prof and calib may be NULL. */
int some_forward(const some_model* model, const some_workspace* ws, int M, int B, const int32_t* cu_frames,
                 int max_frames, int head, some_profiler* prof, some_calibration* calib, cudaStream_t stream);

/* ---- some_forward_f32: the same trunk with fp32 operands on the CUDA cores (no tensor cores, no bf16, exact expf-based
 * activations): the VALIDATION mode behind the "within 1e-3 fp32" line of the contract.  The reference inference path is fp32
 * (inference/me_infer.py:65-76; pl_trainer_precision only affects training).  ~100x slower than some_forward; a checker, not a
 * fallback: the product path never calls it.  Weights are the checkpoint's own fp32 tensors in nn.Linear layout [N, K]
 * (to_q | to_kv concatenated, pointwise convs squeezed, depthwise taps [31][512] with BatchNorm folded, GLU producers NOT
 * row-packed: first half = out, second half = gate). */
typedef struct {
  const float* ln_g[5];
  const float* ln_b[5];
  const float* ffn_w1[2];
  const float* ffn_b1[2];
  const float* ffn_w2[2];
  const float* ffn_b2[2];
  const float* w_qkv;
  const float* w_out;
  const float* b_out;
  const float* w_pw1;
  const float* b_pw1;
  const float* w_dw;
  const float* b_dw;
  const float* w_pw2;
  const float* b_pw2;
} some_block_weights_f32;
typedef struct {
  int lay, outdim;
  const float* w_in[2];
  const float* b_in[2];
  const some_block_weights_f32* blocks; /* host array [(lay + 1) * 2], entry 2 i + s */
  const float* const* glu_w;            /* host array [lay * 2]: 2 i + 0 = glu1 (fed by midi), 2 i + 1 = glu2 */
  const float* const* glu_b;
  const float* w_head;
  const float* b_head;
  const float* w_cut;
  float b_cut;
} some_model_f32;
typedef struct {
  float* x[2];         /* f32 [M,512] residual streams */
  float* a[2];         /* f32 [M,512] */
  float* h[2];         /* f32 [M,2048] */
  float* qkv[2];       /* f32 [M,1536] */
  float* g[2];         /* f32 [M,512] */
  float* y[2];         /* f32 [M,1024] GLU pre-activations */
  const float* units;  /* f32 [M,80] log-mel (input: some_mel_logmel out_f32) */
  float* probs;        /* f32 [M,outdim] (output) */
  float* bounds;       /* f32 [M] (output) */
} some_workspace_f32;
int some_forward_f32(const some_model_f32* model, const some_workspace_f32* ws, int M, int B, const int32_t* cu_frames,
                     int max_frames, int head, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SOME_B200_H_ */
