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

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SOME_B200_VERSION 202

#ifndef __CUDA_RUNTIME_H__
typedef struct CUstream_st* cudaStream_t;
#endif

/* Model geometry the kernels are specialised for (all shipped configs under configs/). */
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
 *   optional per-frame outputs (may be NULL: then they live in the scratch): frame2item i32 [M] (1-based note index of each
 *     frame within its clip, infer_utils.py:27-39), values f32 [M] (phase A's pitch value), rest u8 [M] (phase A's rest
 *     flag); the notes are the same with or without them.  The session's frame curves (some_notes_get_frames) are these.
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

/* ---- K-eval: the validation losses and MIDI accuracy of the training tasks (training/me_task.py:72-154, continuous;
 * training/me_quant_task.py:43-120, quantized) for B labelled clips in one launch, one CTA per clip, without materialising
 * the [M, N] target.  Per clip b (frames [cu_frames[b], cu_frames[b+1]), T = their number):
 *   midi_loss[b]   continuous: sum over T x N of BCEWithLogits(logit, gaussian-blurred target of the collater, me_task.py:26-49),
 *                  max(x,0) - x*y + log1p(exp(-|x|)); quantized: sum over T of CrossEntropy(logits row, note class) with a
 *                  stable log-softmax (every frame has a class: unit2note > 0, so ignore_index never applies)
 *   bound_loss[b]  sum over T of |cumsum(bounds) / sqrt(T) - cumsum(gt) / sqrt(T)|, gt = diff(unit2note, prepend 0) > 0
 *                  (BinaryEMDLoss, modules/losses/bound_loss.py:6-19; the bounds prefix is accumulated in double and rounded
 *                  to float per frame like ATen's CPU cumsum)
 *   correct[b]     frames where MIDIAccuracy(tolerance=0.5).update (modules/metrics/midi_acc.py:16-35) counts a hit:
 *                  neither the prediction nor the label is a rest and |midi_pred - midi_gt| <= 0.5; the prediction is the
 *                  validation step's decode of the activated head (continuous: gaussian-blurred decode, rest = max < threshold;
 *                  quantized: argmax, rest = 128).  The total is T.
 * The sums are the caller's to divide (T * N, T, T).  Reductions run in a fixed order (frame-strided warps, then warps in
 * order) with no atomics: a clip's results do not depend on the other clips of the launch.
 *   logits     f32 [M, N] raw head (SOME_EPI_BIAS_F32), bounds f32 [M] (sigmoid, as the trunk writes them)
 *   unit2note  i32 [M], 1-based note index within the clip, in [1, cu_notes[b+1] - cu_notes[b]]
 *   cu_notes   i32 [B+1]; note_midi f32 (continuous: MIDI with rests interpolated; quantized: class 0..128, rest = 128),
 *              note_rest u8 (continuous only), both [cu_notes[B]]
 *   head       SOME_EVAL_HEAD_TC: sigmoid / softmax exactly as the tensor-core GEMM's head epilogues compute them (some_forward);
 *              SOME_EVAL_HEAD_F32: as the fp32 validation path's head kernel computes them (some_forward_f32)
 *   probs      optional f32 [M, N] (may equal logits): the activated head, bit-identical to what the chosen forward would
 *              have written with the sigmoid / softmax head, for some_decode_notes
 * A frame whose unit2note is out of range makes its clip's three results NaN / -1. */
enum { SOME_EVAL_HEAD_TC = 0, SOME_EVAL_HEAD_F32 = 1 };
typedef struct {
  const float* logits;
  const float* bounds;
  const int32_t* cu_frames;
  const int32_t* unit2note;
  const int32_t* cu_notes;
  const float* note_midi;
  const uint8_t* note_rest;
  int B, M, N;
  int quantized;
  int head;
  float vmin, vmax, deviation, threshold; /* midi_min, midi_max, midi_prob_deviation, rest_threshold */
  double* midi_loss;
  double* bound_loss;
  int32_t* correct;
  float* probs;
} some_eval_args;
int some_eval_clips(const some_eval_args* args, cudaStream_t stream);

/* ---- K-rms (row §8f-1, the step in front of the path): short-time RMS for the silence slicer.
 * Replaces get_rms (utils/slicer2.py:5-38) as called by Slicer.slice (slicer2.py:81): zero padding of frame_length / 2 on
 * both sides, frames of frame_length samples every hop samples, sqrt(mean(x^2)) in float32 with numpy's pairwise summation
 * order, i.e. BIT-identical to the reference so the host state machine (slicer2.py:84-133) cuts identical chunks.
 * wave: device f32 [n_samples] (the whole recording, resident; the chunks are later processed in place);
 * rms: device f32 [n_frames], n_frames = 1 + (n_samples + 2 * (frame_length / 2) - frame_length) / hop. */
int some_slicer_rms(const float* wave, long long n_samples, int frame_length, int hop, float* rms, int n_frames,
                    cudaStream_t stream);
/* The same frames [f_begin, f_end) of a recording of which the buffer holds samples [base, base + held): wave[s - base] is
 * sample s; rms[f - f_begin] receives frame f.  n_samples: the recording's length, or -1 while it is not known (every frame
 * must then read samples before base + held only).  The buffer must hold every sample inside the recording the frames read.
 * Bit-identical to some_slicer_rms on the whole recording. */
int some_slicer_rms_window(const float* wave, long long base, long long held, long long n_samples, int frame_length, int hop,
                           float* rms, long long f_begin, long long f_end, cudaStream_t stream);
/* Many frame windows in one launch (the streams of one some_stream_push_many call).  Window i is the call
 * some_slicer_rms_window(w[i].wave, ..., w[i].f_end) and gets its bits.  Two steps, so that the descriptors can travel in a
 * host-to-device copy the caller makes anyway:
 *   some_slicer_rms_windows_pack  checks every window as some_slicer_rms_window does (the message names the window) and
 *                                 writes the kernel's descriptors to `desc`, host memory of some_slicer_rms_windows_bytes(K) bytes;
 *   some_slicer_rms_windows       launches, sized by the host copy `desc`, reading the descriptors from `desc_d`, a device
 *                                 copy of the same bytes (16-byte aligned) that is in place when the launch runs. */
typedef struct {
  const float* wave;
  long long base, held, n_samples;
  int frame_length, hop;
  float* rms;
  long long f_begin, f_end;
} some_rms_window;
long long some_slicer_rms_windows_bytes(int K);
int some_slicer_rms_windows_pack(const some_rms_window* w, int K, void* desc);
int some_slicer_rms_windows(const void* desc, const void* desc_d, cudaStream_t stream);

/* ---- K-resample (the step in front of the slicer): librosa.resample(y, orig_sr, target_sr, res_type='kaiser_best') as
 * librosa.load calls it (infer.py:34, batch_infer.py:51, webui.py:47; librosa<0.10 -> resampy.resample(filter='kaiser_best')
 * + fix_length), BIT-identical to resampy's float32 loop (float64 taps and products, a float32 rounding after every add, no
 * FMA; restated in oracle/resample.py).  B recordings that share one rate pair, in one launch:
 *   x        f32 mono recordings at sr_orig, recording b = x[x_start[b] .. x_start[b] + x_len[b])  (x_start, x_len int64 [B])
 *   y        f32 outputs at sr_new, recording b = y[y_start[b] ..) (y_start int64 [B]), ceil(x_len[b] * ratio) samples each with
 *            ratio = (double)sr_new / sr_orig; samples from resampy's n_out = floor(x_len[b] * sr_new / sr_orig) on are 0
 *            (librosa.load raises for a recording with n_out < 1: that check is the caller's)
 *   max_out  max_b ceil(x_len[b] * ratio) (grid sizing)
 *   win      f64 [nwin]: the interpolation table, 512 entries per zero crossing (kaiser_best: 32769 entries), already multiplied
 *            by ratio when ratio < 1, as resampy does
 * Downsampling by more than about 11x is rejected (the input window of a tile no longer fits in shared memory). */
int some_resample_kaiser(const float* x, const int64_t* x_start, const int64_t* x_len, float* y, const int64_t* y_start, int B,
                         long long max_out, int sr_orig, int sr_new, const double* win, int nwin, cudaStream_t stream);
/* The same resampling of ONE recording whose input arrives in pieces, by absolute positions: x[i - x_first] is input sample i
 * (x holds [x_first, received)), y[t - y_first] receives output t, for t in [t_begin, t_end).  final = 0: the recording may
 * go on, and only outputs whose right wing ends within the received input are computed (t_end up to the plan's);
 * final != 0: the recording is `received` samples long and outputs up to ceil(received * ratio) include fix_length's zeros.
 * Bit-identical to some_resample_kaiser on the whole recording.
 * some_resample_window_plan: *t_end = the outputs [0, *t_end) that `received` input samples fix, *x_first = the first input
 * sample the outputs from t_begin on read (what a host must keep).  Host only. */
int some_resample_kaiser_window(const float* x, long long x_first, long long received, int final, float* y, long long y_first,
                                long long t_begin, long long t_end, int sr_orig, int sr_new, const double* win, int nwin,
                                cudaStream_t stream);
int some_resample_window_plan(long long received, int final, long long t_begin, int sr_orig, int sr_new, int nwin,
                              long long* t_end, long long* x_first);
/* Many windows in one launch, each with its own recording, rate pair and table: window i is the call
 * some_resample_kaiser_window(w[i].x, ..., w[i].nwin) and gets its bits.  The grid lays the windows' tiles end to end; the
 * dynamic shared memory is the largest the windows' rate pairs need.  Packed and launched in two steps like
 * some_slicer_rms_windows: some_resample_windows_pack checks every window as some_resample_kaiser_window does (the message
 * names the window) and writes the descriptors to host memory of some_resample_windows_bytes(K) bytes;
 * some_resample_kaiser_windows launches from the host copy `desc` and its device copy `desc_d` (16-byte aligned). */
typedef struct {
  const float* x;
  long long x_first, received;
  int final;
  float* y;
  long long y_first, t_begin, t_end;
  int sr_orig, sr_new;
  const double* win;
  int nwin;
} some_resample_window;
long long some_resample_windows_bytes(int K);
int some_resample_windows_pack(const some_resample_window* w, int K, void* desc);
int some_resample_kaiser_windows(const void* desc, const void* desc_d, cudaStream_t stream);

/* ---- K-flac (the step in front of K-resample): the FLAC decode of librosa.load (soundfile -> libsndfile -> libFLAC) for
 * many recordings in one set of launches, from slices of one device byte buffer `data` (restated in oracle/flac.py).
 * Streams with more than 24 bits per sample are the caller's to refuse; so is parsing the metadata blocks.
 *   streams  device [n_streams], sorted by audio_start, disjoint: recording s's frames lie in [audio_start, end) of data
 *            and must agree with its STREAMINFO channels, bps and max block size.
 * some_flac_scan: every byte position of every recording's audio range where a frame header starts that is syntactically
 * valid, has a correct CRC-8 and agrees with the STREAMINFO is a candidate; *count (device int) = their number, and the
 * first min(count, capacity) are written to frames[] in byte order with pos, number, stream, blocksize, header_len,
 * chan_code, variable filled.  Each written candidate is then parsed (subframe syntax, zero padding, CRC-16): status =
 * SOME_FLAC_OK and end = one past its CRC-16, or another status and end = the byte where the problem was found.  A
 * candidate never reads outside its recording's range.  If count > capacity, the call must be repeated with a larger
 * capacity.  workspace: some_flac_scan_workspace_bytes(n_bytes) bytes of device memory.
 * some_flac_decode: decodes frames[chain[k]] (k < n_chain, each parsed OK) into scratch[scratch_off[k] ..] as int32
 * [channels][blocksize], then writes x * 2^-(bps-1) to out: mono (out[out_off[k] + i], np.mean's float32 order over the
 * channels) or interleaved (out[(out_off[k] + i) * channels + c]).  *status (device int, zero on entry) is set if a
 * chained frame fails to decode. */
enum {
  SOME_FLAC_OK = 0,
  SOME_FLAC_TRUNCATED = 1,           /* the frame runs past the end of its recording */
  SOME_FLAC_BAD_CRC16 = 2,
  SOME_FLAC_BAD_PADDING = 3,         /* a subframe's zero bit or the frame's byte-alignment bits are not 0 */
  SOME_FLAC_RESERVED_SUBFRAME = 4,   /* reserved subframe type or FIXED order > 4 */
  SOME_FLAC_BAD_WASTED_BITS = 5,     /* wasted bits >= the subframe's bits per sample */
  SOME_FLAC_BAD_ORDER = 6,           /* predictor order > block size */
  SOME_FLAC_BAD_LPC = 7,             /* LPC precision code 1111 or negative shift */
  SOME_FLAC_BAD_RESIDUAL = 8,        /* reserved residual coding method */
  SOME_FLAC_BAD_PARTITION = 9        /* partition order does not divide the block, or its first partition < order */
};
typedef struct {
  int64_t audio_start;
  int64_t end;
  int32_t channels, bps, max_blocksize, reserved;
} some_flac_stream;
typedef struct {
  int64_t pos;                       /* byte offset of the frame header in data */
  int64_t number;                    /* coded frame number (fixed blocking) or first sample number (variable blocking) */
  int64_t end;
  int32_t stream;
  int32_t blocksize;
  int16_t header_len;
  uint8_t chan_code;                 /* 0-7 independent channels, 8 left/side, 9 side/right, 10 mid/side */
  uint8_t variable;                  /* blocking strategy bit */
  int32_t status;
} some_flac_frame;
uint64_t some_flac_scan_workspace_bytes(long long n_bytes);
int some_flac_scan(const uint8_t* data, long long n_bytes, const some_flac_stream* streams, int n_streams,
                   some_flac_frame* frames, int capacity, int* count, void* workspace, cudaStream_t stream);
int some_flac_decode(const uint8_t* data, const some_flac_stream* streams, const some_flac_frame* frames, const int32_t* chain,
                     const int64_t* scratch_off, const int64_t* out_off, int n_chain, int32_t* scratch, float* out, int mono,
                     int* status, cudaStream_t stream);
/* some_flac_chain (host, no CUDA call): the frames a sequential decoder walks, from the candidate list of some_flac_scan
 * (frames[0 .. n_frames), in byte order, downloaded to the host).  Recording r starts its walk at recs[r].audio_start; each
 * next frame starts where the current one ends and carries the next frame number (fixed blocking) or sample number (variable
 * blocking); the walk stops after recs[r].length samples (STREAMINFO; 0 = not stated: at recs[r].end).  Byte offsets in the
 * messages are counted from recs[r].base (the first byte of the recording's file in `data`).  Writes the chained indices of
 * recording r to chain[first[r] .. first[r + 1]) (first: [n_recs + 1]; capacity n_frames always suffices) and its decoded
 * length to lengths[r].  Refused, with *failed = r and a message that names no file, when a header is missing where a frame
 * must start, a chained frame's status is not SOME_FLAC_OK, a frame or sample number leaves a gap or overlaps or the blocking
 * strategy changes, a frame decodes past the STREAMINFO length, or the recording ends early. */
typedef struct {
  int64_t base, audio_start, end, length;
} some_flac_range;
int some_flac_chain(const some_flac_frame* frames, int n_frames, const some_flac_range* recs, int n_recs, int32_t* chain,
                    int capacity, int64_t* first, int64_t* lengths, int* failed);
/* some_flac_chain_resume (host, no CUDA call): the same walk for one recording whose bytes arrive in pieces, continued over
 * the candidates of one window at a time.  `walk` keeps what the walk needs between windows: pos (the file offset where the
 * next frame must start; set it to the first frame byte, with the rest zero and strategy -1, before the first window), the
 * samples and frames chained so far, the blocking strategy and whether the walk is done.  The window holds the file's bytes
 * from walk->pos on: file offset x is x + base in the candidates' coordinates, and the window ends at `stop`.  Writes the
 * indices of the frames it chains to chain[0 .. *n_chained).  final != 0: the window runs to the end of the file, and every
 * check of some_flac_chain applies with its message (offsets from the file's first byte).  Before that, the walk stops
 * without error at a frame that is SOME_FLAC_TRUNCATED (the window ends inside it) or where fewer than 16 bytes (the
 * longest frame header) follow and no header was found; the next window starts at walk->pos. */
typedef struct {
  int64_t pos, got, count;
  int32_t strategy, done;
} some_flac_walk;
int some_flac_chain_resume(const some_flac_frame* frames, int n_frames, int64_t base, int64_t stop, int64_t length, int final,
                           some_flac_walk* walk, int32_t* chain, int capacity, int* n_chained);

/* ---- Container metadata on the host (csrc/audio_host.cu, no CUDA call): what some_b200.audio.load accepts, but for one
 * kind of file: integer PCM in 5-8 byte containers, which scipy reads as int64 and audio.decode_wav scales by 2^-63, is
 * refused here (and with it 1-8 bit PCM in containers wider than one byte, which scipy misreads).
 * some_audio_info  RIFF/WAVE as scipy.io.wavfile.read walks it (fmt tag 1: PCM in 1, 2, 3 or 4 byte containers; tag 3: float32
 *                  or float64; tag 0xFFFE with a PCM or float subformat; any number of channels; other chunks skipped with
 *                  their pad byte; a data chunk cut short by the end of the file yields the whole frames present), or fLaC,
 *                  optionally behind an ID3v2 tag (the first block a 34-byte STREAMINFO, type 127 invalid; up to 24 bits per
 *                  sample), or FORM/AIFF and FORM/AIFC as libsndfile reads them (COMM before SSND, other chunks skipped
 *                  with their pad byte, the walk bounded by the FORM size and ending with the SSND chunk; the rate is the
 *                  integer part of COMM's 80-bit extended value; the frames are the whole frames of the SSND bytes within
 *                  its stated size and the file; integer PCM of 1-32 bits big-endian or `sowt`, `raw ` 8-bit unsigned,
 *                  `fl32` / `fl64` big-endian float, `ulaw` / `alaw` G.711).  Refused with a reason (audio.decode_wav's, i.e.
 *                  scipy's, text for the WAV walk; one naming FLAC; "AIFF/IFF: ..." for AIFF) and the byte offset:
 *                  other containers (Ogg, MP3, RIFX, RF64, CAF, AU) by name (after an ID3v2 tag also with the byte offset
 *                  where the fLaC marker was looked for), truncated or missing chunks, unsupported tags,
 *                  compression types or sample sizes, a bad STREAMINFO, an AIFF rate outside [1, 2^31). */
enum { SOME_AUDIO_WAV = 1, SOME_AUDIO_FLAC = 2, SOME_AUDIO_AIFF = 3 };
/* Sample containers: little-endian U8 .. F64 (WAV, AIFF-C `sowt` and `raw `), and for AIFF: S8 (1-8 bit signed), the
 * big-endian S16BE .. F64BE and G.711 ULAW / ALAW (one byte per sample). */
enum { SOME_PCM_U8 = 1, SOME_PCM_S16 = 2, SOME_PCM_S24 = 3, SOME_PCM_S32 = 4, SOME_PCM_F32 = 5, SOME_PCM_F64 = 6,
       SOME_PCM_S8 = 7, SOME_PCM_S16BE = 8, SOME_PCM_S24BE = 9, SOME_PCM_S32BE = 10, SOME_PCM_F32BE = 11, SOME_PCM_F64BE = 12,
       SOME_PCM_ULAW = 13, SOME_PCM_ALAW = 14 };
typedef struct {
  int container;                 /* SOME_AUDIO_* */
  int rate, channels, bits;      /* bits: the fmt chunk's bits per sample / STREAMINFO's / COMM's sampleSize */
  int kind;                      /* WAV, AIFF: SOME_PCM_* (the sample container); FLAC: 0 */
  int min_blocksize, max_blocksize;   /* FLAC STREAMINFO; WAV, AIFF: 0 */
  int reserved;
  long long frames;              /* samples per channel (FLAC: STREAMINFO's, 0 = not stated) */
  long long data_offset;         /* WAV, AIFF: first sample byte; FLAC: first frame byte (after the metadata blocks) */
  long long data_bytes;          /* WAV, AIFF: frames * channels * sample bytes; FLAC: to the end of the data */
} some_audio_meta;
int some_audio_info(const void* data, long long n_bytes, some_audio_meta* out);
/* some_audio_walk: the walk of some_audio_info fed in pieces; some_audio_info is the case where all bytes come in one feed with
 * end != 0.  A feed costs time in proportion to its own bytes, and the walker holds no skipped bytes (ID3 tags, metadata
 * blocks other than STREAMINFO, WAV and AIFF chunks other than fmt, data, COMM and SSND, the AIFF-C compression name) and no
 * audio: *held (may be NULL) stays within 48 bytes.
 * After each feed: -1 with some_audio_info's message and offset for the same bytes (or for the whole file) once the refusal
 * is certain; else 0 and *known = 1 once the metadata is in *meta (WAV, AIFF: from the data / SSND chunk's header, with its
 * stated size; FLAC: after the last metadata block; final after the end), and the audio bytes of this feed are the file
 * offsets [*audio_begin, *audio_end): WAV / AIFF sample bytes of the whole frames within the data / SSND chunk's stated size,
 * FLAC everything after the metadata.  The rules that depend on where the file ends (a data or SSND chunk cut short keeps its
 * whole frames, a partial 24-bit sample or multi-channel WAV frame is refused, "Unexpected end of file", chunks after the
 * data chunk) apply at the feed with end != 0.  AIFF reads the same in both modes: its COMM chunk must come before SSND (an
 * SSND chunk before COMM is refused when its header is reached) and nothing after the SSND chunk is read.
 *   stream != 0: a second WAV data chunk, or a fmt chunk after the data chunk, is refused when its header is reached; without
 * it (and in some_audio_info) the last data chunk is read with the last fmt chunk, as scipy reads them. */
typedef struct some_audio_walk some_audio_walk;
int some_audio_walk_create(int stream, some_audio_walk** out);
int some_audio_walk_feed(some_audio_walk* w, const void* data, long long n_bytes, int end, int* known, some_audio_meta* meta,
                         long long* audio_begin, long long* audio_end, long long* held);
int some_audio_walk_destroy(some_audio_walk* w);

/* ---- K-pcm: the samples of RIFF/WAVE data chunks and AIFF / AIFF-C SSND chunks as libsndfile hands them to librosa.load,
 * many recordings in one launch.  u8 -> (x - 128) / 128, s8 / s16 / s24 / s32 (either byte order) -> x / 2^(bits - 1) of
 * the container (s32 rounded to float32 first, as numpy's astype), f32 as is, f64 rounded to nearest float32 (either byte
 * order), G.711 u-law / A-law -> the 16-bit value of the standard expansion / 32768.  Samples may start at any byte.  Each
 * kind's container is 1 (u8, s8, u-law, A-law), 2, 3, 4 (s32, f32) or 8 bytes.  mono != 0: out[i] = np.mean's float32 order over
 * librosa's (channels, n) view (channels added one after another below 8, numpy's 8-way pairwise sum from 8 to 128 channels,
 * then / channels; the FLAC emitter uses the same function); mono == 0: interleaved out[i * channels + c].
 * Packed and launched in two steps like some_slicer_rms_windows: some_pcm_decode_pack checks every item (the message names
 * it; mono needs channels <= 128) and writes the descriptors to host memory of some_pcm_decode_bytes(K) bytes; some_pcm_decode
 * launches from the host copy `desc` and its device copy `desc_d` (16-byte aligned). */
typedef struct {
  const uint8_t* data;           /* device: the first byte of the first sample */
  long long frames;              /* samples per channel */
  int channels, kind, mono, reserved;
  float* out;                    /* device: frames floats (mono) or frames * channels */
} some_pcm_item;
long long some_pcm_decode_bytes(int K);
int some_pcm_decode_pack(const some_pcm_item* items, int K, void* desc);
int some_pcm_decode(const void* desc, const void* desc_d, cudaStream_t stream);

/* ---- K-downmix (csrc/downmix.cu): librosa.to_mono of float32 audio already in device memory, many recordings in one launch.
 * Output sample f of an item is np.mean(y, axis=0) in float32 of librosa's (channels, frames) view y, bit for bit.  numpy's
 * order depends on the layout:
 *   SOME_DOWNMIX_MONO         a one-dimensional recording (one channel): the value itself;
 *   SOME_DOWNMIX_PLANAR       frames contiguous, channel c at data + c * channel_stride (>= frames): the channels added in
 *                             order starting from +0.0 (an all -0.0 frame gives +0.0), then / channels;
 *   SOME_DOWNMIX_INTERLEAVED  channels contiguous, frame f at data + f * channels: numpy's pairwise sum, the order of
 *                             some_pcm_decode's mono output; an item of one frame reads channel c at data + c * channel_stride
 *                             (numpy reduces a lone frame in this order whatever its strides).
 * some_downmix_layout names the layout of `channels` x `frames` floats with the given strides in floats (channel_stride 0 with
 * one channel: a one-dimensional recording), or refuses any other stride pattern (host only, no CUDA call).  Packed and
 * launched like some_pcm_decode: some_downmix_pack checks every item (the message names it) into host memory of
 * some_downmix_bytes(K) bytes; some_downmix launches from it and its device copy desc_d (16-byte aligned).  The native session
 * down-mixes device audio with the same launch (some_session_transcribe_device). */
enum { SOME_DOWNMIX_MONO = 0, SOME_DOWNMIX_PLANAR = 1, SOME_DOWNMIX_INTERLEAVED = 2 };
typedef struct {
  const float* data;             /* device: channel 0 of frame 0 */
  long long frames;              /* samples per channel */
  int channels;                  /* 1..128 */
  int layout;                    /* SOME_DOWNMIX_* */
  long long channel_stride;      /* floats between channels: planar, and an interleaved item of one frame */
  float* out;                    /* device: frames floats */
} some_downmix_item;
int some_downmix_layout(int channels, long long frames, long long channel_stride, long long frame_stride, int* layout);
long long some_downmix_bytes(int K);
int some_downmix_pack(const some_downmix_item* items, int K, void* desc);
int some_downmix(const void* desc, const void* desc_d, cudaStream_t stream);

/* ---- MIDI bytes (host, no CUDA call): the Standard MIDI File some_b200.midi.build_midi_file(offsets, segments,
 * tempo).to_bytes() writes, with note_dur seconds = (double)note_dur * timestep.  Chunk c holds notes
 * [sum counts[0 .. c), + counts[c]).  Ticks follow infer_utils.build_midi_file: offsets * tempo * 8 rounded half to even,
 * each chunk's note ends from np.round of the float64 cumulative duration times tempo * 8, notes clipped at the next chunk's
 * tick, rests and empty notes skipped.  *size = the bytes of the file; they are written only when capacity >= *size (buf may
 * be NULL with capacity 0, to ask for the size).  Refused where Python raises (a note outside 0..127 after rounding, a negative
 * delta time) and for a tempo whose round(60e6 / bpm) does not fit the 24 bits of set_tempo.
 * some_notes_midi (below, with the session) does the same for a session's result. */
int some_midi_write(int n_chunks, const double* offsets, const int32_t* counts, const float* note_midi, const int32_t* note_dur,
                    const uint8_t* note_rest, double timestep, double tempo, uint8_t* buf, size_t capacity, size_t* size);

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
/* some_forward_f32_tiled: the same launch sequence and arguments, with register- and shared-memory-tiled fp32 GEMM, attention
 * and depthwise-conv kernels that keep every output's operation order: every buffer of `ws` (x a h qkv g y probs bounds)
 * holds the same bits as after some_forward_f32, at many times its speed: the fp32 precision of Engine.infer and of an
 * fp32 session.  Every workspace buffer and GEMM operand must be 16-byte aligned, with K and row pitches multiples of 4
 * floats (true for every buffer some_workspace_f32_carve hands out and every tensor of the model); otherwise the call fails
 * with an error and launches nothing.  A clip's rows do not depend on the other clips of the launch. */
int some_forward_f32_tiled(const some_model_f32* model, const some_workspace_f32* ws, int M, int B, const int32_t* cu_frames,
                           int max_frames, int head, cudaStream_t stream);
/* Size of, and carving of one 256-byte aligned device block into, an fp32 workspace for M rows: x a h qkv g y, units, probs,
 * bounds in that order, each 256-byte aligned. */
uint64_t some_workspace_f32_bytes(int M, int outdim);
int some_workspace_f32_carve(void* device_block, uint64_t bytes, int M, int outdim, some_workspace_f32* ws);

/* ---- Native inference session (csrc/session.cu): the export/deployment path of the reference (export.py + deployment/) for
 * hosts without Python.  `python -m some_b200.export --model CKPT` writes a checkpoint, its load-time bias correction applied
 * (Engine.calibrate), into one self-contained model file (format: INTEGRATION.md "Deploying without Python"); a session opens
 * that file and transcribes recordings with the kernels above, enqueued in the order of some_b200/engine.py, so its notes are
 * bit-identical to plugin.infer() / Engine.infer_sliced.  Host memory in, host memory out; the session owns its streams and
 * buffers.  Several threads may share a session, each with its own result: calls that queue while a step runs are run
 * together as one GPU step (see "Calls from several threads" below).
 *
 * some_session_open       reads and validates the whole file before any CUDA call (magic, format version, ABI, directory
 *                         bounds, every tensor present with the shape implied by lay / outdim, file size); refuses a device
 *                         that is not sm_90; uploads the weights.  < 0 on failure, some_last_error() names the file and problem.
 * some_session_transcribe B mono float32 clips at the model's sample rate -> one entry per clip in `out`, in input order.  The
 *                         clips are staged through pinned memory; the upload of each pipeline chunk overlaps the kernels of
 *                         the previous one (Engine.enqueue).  Clips are independent: results do not depend on the batch.
 * some_session_transcribe_sliced
 *                         one mono recording at any integer rate (resampled on the device as librosa.load does when the rate
 *                         differs; too-short inputs are refused as resampy does), cut by the silence slicer (params NULL:
 *                         Slicer(sr, max_sil_kept=1000) as in infer.py) and transcribed where it lies: one entry per chunk,
 *                         with its sample range in the (resampled) recording.
 * some_notes_get          a clip's notes: note_midi f32, note_dur in frames (seconds = dur * timestep, the float64 product of
 *                         me_infer.py:95), note_rest u8; the pointers stay valid until the next call that fills `n`. */
typedef struct some_session some_session;
typedef struct some_notes some_notes;
typedef struct {
  int sample_rate, hop, outdim, quantized, bias_corrected;
  double timestep; /* hop / sample_rate */
} some_session_info;
/* Slicer constructor arguments (utils/slicer2.py), in milliseconds / dB like Slicer(sr, threshold, min_length, min_interval,
 * hop_size, max_sil_kept) */
typedef struct {
  double threshold_db, min_length_ms, min_interval_ms, hop_size_ms, max_sil_kept_ms;
} some_slicer_params;
/* ... and the frame counts Slicer derives from them (Python's round, half to even) */
typedef struct {
  float threshold; /* 10^(dB / 20) rounded to float32: `rms < threshold` compares in float32 */
  int hop_size, win_size, min_length, min_interval, max_sil_kept;
} some_slicer_frames;

int some_session_open(const char* path, int device, some_session** out);
/* ---- One session on several devices: a replica of the model on each listed device, the chunks of every call spread over them.
 * For every call, a session opened on devices [d0, d1, ...] returns exactly what a session on [d0] returns: the same clips and
 * chunks in the same order, the same ranges and bit-identical notes (a chunk's notes do not depend on the rest of its batch).
 * The front end (byte upload, FLAC scan and decode, PCM decode, resampling, RMS windows, the slicer, the stream buffers) runs
 * on d0 as in a one-device session; the chunks of the call are then assigned with some_shard_clips, replica 0 runs its share
 * on the calling thread and each other replica its share on a thread of its own (created at open, joined at close), with the
 * caller's some_set_pdl setting.  Chunks on d0's device go to replica r with cudaMemcpyPeerAsync (peer access is used when
 * the application has enabled it, not required); host clips of some_session_transcribe are staged straight to their replica.
 *   Each replica holds its own copy of the weights (104 MB for two_head, 235 MB for midi_conformer) and the workspace of its
 * share.  A device may be listed twice: two replicas on one GPU.
 *   some_session_open_devices checks, in this order: the arguments (devices not NULL, 1 <= n <= 64, every entry >= 0), the
 * model file exactly as some_session_open does, before any CUDA call, then every listed device (it exists and is sm_90)
 * before anything is allocated; a refused device is named by its index in the list.  some_session_open(path, d, out) is the
 * n == 1 case.  A device error on any replica fails the call with a message naming the device; every replica's streams are
 * waited for and the session stays usable.  some_session_close waits for every replica and frees each one's memory on its own
 * device. */
int some_session_open_devices(const char* path, const int* devices, int n, some_session** out);
/* The session's devices in replica order: *n = their count, the first min(capacity, *n) written to devices. */
int some_session_get_devices(const some_session* s, int* devices, int capacity, int* n);
/* For each replica, the chunks and frames (1 + samples / 512 each) it ran in the session's last completed step (with one
 * calling thread: its last completed call): *n = the replica count, the first min(capacity, *n) written. */
int some_session_get_load(const some_session* s, int64_t* chunks, int64_t* frames, int capacity, int* n);
/* ---- Calls from several threads.  Every call that reaches the GPU (every session and stream call below, after the checks it
 * makes before any GPU work) becomes a request in a first-in, first-out queue of the session.  If no step is running, the
 * calling thread runs the next step itself: the oldest request and every later queued request that may join it, in arrival
 * order, as one GPU step; it hands each request its result, and repeats while its own request has not run.  Meanwhile the
 * other callers wait for their own request.  There is no waiting window: a lone caller, or a single-threaded host, runs the
 * same steps as before, and calls merge only when they queue behind a running step.
 *   Which requests may share a step: clip calls (some_session_transcribe) with clip calls; sliced and encoded calls together
 * (one recordings step: their recordings decoded, resampled, cut and transcribed as one); PCM stream calls together (push,
 * finish, push_many: one stream step); encoded stream calls together (push_bytes*, finish of an encoded stream); peeks
 * together (some_stream_peek*: one batch of open regions).  Calls of
 * different kinds run as consecutive steps.  Never in one step: two requests that touch the same some_stream or the same
 * some_notes (the later one waits for a later step, so each stream's calls apply in arrival order), or requests whose threads
 * have different some_set_pdl settings (the step runs with its requests' setting).  A request joins only while the step's
 * model-rate samples stay within max(the oldest request's own, SOME_SESSION_STEP_SAMPLES), so a merged step holds no more
 * device memory than its largest request alone or a step of that size.  The samples are known before any GPU work: clips,
 * the sliced and encoded recordings at the model's rate, a PCM stream push's samples at the model's rate, and an encoded
 * stream push's bytes, and a peek's open regions.  An encoded call with a FLAC file that states no length (STREAMINFO total 0) takes no joiners and joins
 * no step.  A request that cannot join stays the oldest, and the next step is built around it.
 *   Results: a step of several requests gives each request exactly what it gives alone (a chunk's notes do not depend on the
 * rest of its batch).  An encoded call refused after the scan (a corrupt FLAC file) fails alone with the message and item
 * index it gives alone and no out[i] written, and a refused encoded stream fails only its own call; the other requests of the
 * step run on.  Each caller's some_last_error() is set on its own thread.  A device error fails every request of its step
 * with the device's message, and the session stays usable. */
#define SOME_SESSION_STEP_SAMPLES 84672000LL /* 64 recordings x 30 s at 44.1 kHz: about 4.5 GB of activations */
typedef struct {
  int64_t calls;     /* requests queued since open */
  int64_t steps;     /* steps run since open */
  int64_t max_calls; /* the most requests one step has held */
  int64_t queued;    /* requests waiting at this moment (not counting those of a step in progress) */
} some_session_stats;
int some_session_get_stats(const some_session* s, some_session_stats* stats);
/* Host only, no CUDA call: owner[i] = the replica of clip i of n.  Longest processing time first: clips in order of
 * (-cost, index), cost = T * (103.31e6 + 16384 * T) with T = 1 + lens[i] / 512, each to the least loaded replica (ties: the
 * lowest).  The sessions above and some_b200.dist.shard_clips assign clips with it. */
int some_shard_clips(const int64_t* lens, int n, int replicas, int32_t* owner);
int some_session_close(some_session* s);
int some_session_get_info(const some_session* s, some_session_info* info);
/* The precision of the model file the session opened, which every call runs at: SOME_PRECISION_BF16 (the product trunk,
 * some_forward) or SOME_PRECISION_FP32 (a file written by `python -m some_b200.export --precision fp32`: the checkpoint's fp32
 * tensors, log-mel as f32 and some_forward_f32_tiled, notes bit-identical to Engine.infer(..., precision='fp32')).  The model
 * file records it in the header's int32 at byte 88, which bf16 files leave zero. */
enum { SOME_PRECISION_BF16 = 0, SOME_PRECISION_FP32 = 1 };
int some_session_get_precision(const some_session* s, int* precision);
int some_session_transcribe(some_session* s, const float* const* clips, const int64_t* lens, int B, some_notes* out);
int some_session_transcribe_sliced(some_session* s, const float* samples, long long n, int sample_rate,
                                   const some_slicer_params* params, some_notes* out);
int some_notes_create(some_notes** out);
int some_notes_destroy(some_notes* n);
int some_notes_clips(const some_notes* n); /* number of clips / chunks (< 0: error) */
int some_notes_get(const some_notes* n, int clip, int* count, const float** note_midi, const int32_t** note_dur,
                   const uint8_t** note_rest, int64_t* begin, int64_t* end); /* any output pointer may be NULL */
/* Frame curves: what lies under and between the notes, for pitch-line displays.  Off by default.  While
 * some_notes_set_frames(n, 1) is in effect, every call that fills `n` (transcribe, sliced, encoded, stream push / finish /
 * push_many / push_bytes*, peek*) also fills one curve set per clip or chunk, in the order of the notes; set it before the
 * call, not while a call on `n` runs.  For clip `clip` of T frames (T = 1 + len / hop, len: its samples at the model's rate,
 * the rows the model ran), some_notes_get_frames gives:
 *   midi        f32 [T]  the pitch value of each frame: continuous models, the gaussian-blurred decode of the probabilities
 *                        (decode_gaussian_blurred_probs, utils/infer_utils.py:9-24); quantized models, clip(argmax, 0, 127)
 *                        (me_quant_infer.py:28-31)
 *   rest        u8 [T]   1 where the frame is a rest: max probability < rest_threshold, or argmax == 128 (quantized)
 *   bound       f32 [T]  the boundary probability the model wrote for the frame (sigmoid of its cut head)
 *   note_index  i32 [T]  the 1-based note the frame belongs to (decode_bounds_to_alignment, infer_utils.py:27-39); the notes
 *                        of some_notes_get are exactly the runs of equal note_index, in order
 * Frame t of a clip is centred at sample begin + t * hop of the clip's range (begin from some_notes_get): the mel frames are
 * taken after 1024 + 1024 zero samples of padding with a centre-free STFT (spec.py:48-60).  The notes are bit-identical with
 * frames on or off.  Cost: 13 bytes per frame more in the step's one download, plus one device copy of the bounds per
 * pipeline chunk; a step copies that much more only when one of its results asks for curves.  The pointers stay valid until
 * the next call that fills `n`; any output pointer may be NULL.  Refused: a NULL `n`, a clip out of range, and notes that
 * were last filled with frames off. */
int some_notes_set_frames(some_notes* n, int on);
int some_notes_get_frames(const some_notes* n, int clip, int* frames, const float** midi, const uint8_t** rest,
                          const float** bound, const int32_t** note_index);
/* some_midi_write over a result: chunk offsets begin / sample_rate seconds, as infer.py passes them to build_midi_file. */
int some_notes_midi(const some_notes* n, int sample_rate, double timestep, double tempo, uint8_t* buf, size_t capacity,
                    size_t* size);

/* ---- Encoded files in, notes out: librosa.load(file, sr=None, mono=True) of WAV, FLAC and AIFF files on the GPU, then the
 * slicer and the model.  For item i, out[i] receives what some_session_transcribe_sliced(s, y, n, rate, params, out[i]) gives for
 * y, rate = audio.load(file, sr=None, mono=True): the same chunk ranges (at the model's rate) and bit-identical notes.
 * Results do not depend on the other items of the call.
 *   One GPU step for all items: every item's audio bytes go up in one pinned copy; one some_flac_scan over the FLAC items,
 * one download of its candidates and some_flac_chain on the host; one some_flac_decode and one some_pcm_decode into a
 * native-rate buffer (items at the model's rate are decoded straight into the model-rate buffer); one
 * some_resample_kaiser_windows launch for every item at another rate; one some_slicer_rms_windows launch, one download and
 * one synchronise; the slicer on the host per item; one batch through the model for the chunks of all items.
 *   Device memory held during the call (grow-only, kept by the session): the items' audio bytes, 4 bytes per FLAC sample and
 * channel (the decoder's int32 scratch), 4 bytes per native-rate sample of the items at another rate, 4 bytes per model-rate
 * sample of all items, plus the model's activations for the chunks; the caller bounds it by choosing `count`.  The same bytes
 * are staged in pinned host memory.
 *   Refused before any GPU work, with the index i in the message and no out[i] touched: NULL arrays or count < 0; a NULL or
 * empty item; two entries sharing one some_notes; anything some_audio_info refuses; mono down-mix of more than 128 channels; a
 * rate pair the resampler does not support; a recording too short to resample.  A corrupt FLAC stream is refused after the
 * scan with its index and some_flac_chain's message, and no out[i] is written.  After a device error the session stays
 * usable.  The call is one request (see "Calls from several threads"); count == 0 does nothing.  params NULL: Slicer(sr,
 * max_sil_kept=1000). */
typedef struct {
  const void* data;
  long long n_bytes;
} some_encoded;
int some_session_transcribe_encoded(some_session* s, const some_encoded* items, int count, const some_slicer_params* params,
                                    some_notes* const* out);

/* ---- Labelling a DiffSinger dataset (csrc/label.cu, host only): batch_infer.py's note_seq / note_dur fields of
 * transcriptions.csv, byte for byte as some_b200.batch.row_notes(ph_dur, ph_num, note_timeline(offsets, segments), round_midi)
 * writes them (batch_infer.py:56-81, 84-135, 178-219): the notes on one timeline rounded to 6 decimals, each start clipped at
 * the previous end; word spans from ph_dur / ph_num; note edges within 0.05 s of a word edge snapped to it; per word the
 * touching notes and a rest for any uncovered remainder (round_midi: the note of largest overlap, or rest, for the whole
 * word).  Python's arithmetic is kept where it decides a digit: round(x, 6) on the exact binary value, str(float) as
 * CPython's shortest repr (5e-05, 2.0), CPython 3.12's compensated sum(), int(round(m - round(m), 2) * 100) cents.
 * ph_dur / ph_num are the CSV fields: values separated by single spaces, ph_dur decimal numbers with an optional exponent,
 * ph_num integers; any other form is refused.
 *   some_label_write  chunk c holds notes [sum counts[0 .. c), + counts[c]) starting offsets[c] seconds into the recording;
 *                     note seconds = (double)note_dur * timestep (frames, as me_infer.py:95).  *seq_size / *dur_size = the
 *                     bytes of each field including its terminating NUL; a field is written only when its capacity holds it
 *                     (buffers may be NULL with capacity 0, to ask for the sizes).
 *   some_notes_label  the same over one result of the session (chunk offsets begin / sample_rate, as some_notes_midi). */
int some_label_write(int n_chunks, const double* offsets, const int32_t* counts, const float* note_midi, const int32_t* note_dur,
                     const uint8_t* note_rest, double timestep, const char* ph_dur, const char* ph_num, int round_midi, char* seq_buf,
                     size_t seq_cap, size_t* seq_size, char* dur_buf, size_t dur_cap, size_t* dur_size);
int some_notes_label(const some_notes* n, int sample_rate, double timestep, const char* ph_dur, const char* ph_num, int round_midi,
                     char* seq_buf, size_t seq_cap, size_t* seq_size, char* dur_buf, size_t dur_cap, size_t* dur_size);
/* some_session_label_dataset: the command of batch_infer.py:149-226 (`--dataset DIR [--csv PATH] [--round_midi]
 * [--overwrite]`) as some_b200.batch.batch_infer_dataset runs it with load_audio=audio.load_native; the output file is
 * byte-identical to it, whatever the frame budget and the session's devices.
 *   Reads DIR/transcriptions.csv as csv.DictReader does (UTF-8; the excel dialect: quoted fields, doubled quotes, newlines
 * inside quotes; blank lines skipped; short rows padded with absent fields).  Item `name` is read from DIR/wavs/{name}.wav,
 * whatever format its bytes are (WAV, FLAC, AIFF).  A file that does not exist goes to on_missing(path, user) (may be NULL),
 * in row order, before any GPU work (batch_infer.py prints "WARNING: audio file does not exist: '<path>'"; the library prints
 * nothing), and its row keeps its fields.  The other rows go to some_session_transcribe_encoded in groups of at most
 * params->max_frames frames (1 + samples / hop per item at the model's rate; an item above the budget goes alone; 0 or
 * params NULL: SOME_SESSION_STEP_SAMPLES / hop), with the slicer params->slicer (NULL: Slicer(sr, max_sil_kept=1000)); a
 * worker thread reads the files of the next group while a group's step runs.  Writes csv_path (NULL: DIR/transcriptions.csv)
 * as csv.DictWriter does: the fieldnames name, ph_seq, ph_dur, ph_num, note_seq, note_dur, QUOTE_MINIMAL, \r\n line ends,
 * UTF-8, empty for absent fields.  Paths in messages and on_missing are spelled as pathlib spells them.
 *   Refused before any GPU work, with the output file untouched: an existing output without `overwrite` (the reference's
 * FileExistsError text); a transcriptions.csv that cannot be read or is not UTF-8; when there are rows: a missing name, ph_dur
 * or ph_num column, and columns outside the six fieldnames or rows longer than the header (DictWriter's "dict contains fields
 * not in fieldnames: ..." text, fields in the header's order).  The reference truncates the output to its header line in that
 * last case and raises; here the file is not touched.  A row with audio whose ph_dur / ph_num does not parse is refused, naming
 * the item (the reference raises after transcribing it).  The session is used only when a row has audio (s may be NULL when
 * none has).
 *   A file the encoded step refuses (e.g. a corrupt FLAC stream) or that cannot be read stops the command with the session's
 * message, naming the file; nothing is written.  report (may be NULL) receives the counts and times of a successful call. */
typedef struct {
  const some_slicer_params* slicer; /* NULL: Slicer(sr, max_sil_kept=1000) */
  long long max_frames;             /* frame budget of one group; 0: SOME_SESSION_STEP_SAMPLES / hop */
} some_label_params;
typedef struct {
  int64_t rows;          /* data rows of transcriptions.csv */
  int64_t labelled;      /* rows whose audio was transcribed */
  int64_t missing;       /* rows whose audio file does not exist */
  int64_t groups;        /* some_session_transcribe_encoded calls */
  int64_t chunks;        /* slicer chunks of all labelled items */
  double audio_seconds;  /* of the labelled items (their frames / rate) */
  double seconds;        /* wall time of the call */
  double gpu_seconds;    /* of which inside some_session_transcribe_encoded; the rest is host work the steps did not hide */
} some_label_report;
typedef void (*some_label_missing_fn)(const char* path, void* user);
int some_session_label_dataset(some_session* s, const char* dataset_dir, const char* csv_path, int round_midi, int overwrite,
                               const some_label_params* params, some_label_missing_fn on_missing, void* user,
                               some_label_report* report);
/* The slicer's decisions on the HOST (no CUDA call): some_slicer_derive fills the frame counts for a sample rate (params NULL:
 * the session's defaults); some_slicer_ranges turns the RMS list of a recording of n_samples samples (some_slicer_rms) into the
 * [begin, end) sample ranges of its chunks, ranges[2 k], ranges[2 k + 1] (the cuts of Slicer.slice, utils/slicer2.py:82-145).
 * *count = the number of ranges; capacity n_frames / 2 + 2 always suffices. */
int some_slicer_derive(int sample_rate, const some_slicer_params* params, some_slicer_frames* out);
int some_slicer_ranges(const float* rms, int n_frames, long long n_samples, const some_slicer_frames* frames, int64_t* ranges,
                       int capacity, int* count);

/* The slicer on an RMS list that arrives in pieces (host only, no CUDA call): the same decisions as some_slicer_ranges, each
 * range returned as soon as no later frame can change it.  Both, and some_slicer_derive, are in csrc/slicer.cu next to the
 * RMS kernel; the session and the streams below take their cuts from them.
 * some_slicer_stream_feed    the next n_frames RMS frames; `fixed` = the samples known so far, which must complete those frames
 *                            (frame k reads samples up to k hop_size - win_size / 2 + win_size - 1).  Returns the ranges that
 *                            became final: the range before a cut silent run once the voiced frame after the run is known, or
 *                            once the run has lasted to frame max(ss + 2 max_sil_kept, ss + min_interval - 1,
 *                            chunk begin + min_length - 1) (ss: its first frame), whichever comes first; none while no more
 *                            than min_length * hop_size samples are fixed (a shorter recording is one chunk).
 * some_slicer_stream_finish  the frames not fed yet (those that read past the end) and the final length: the remaining ranges,
 *                            after the trailing-silence and short-recording rules.  No feed after it.
 * some_slicer_stream_keep_from  what a host must keep of the audio: a range not returned yet begins at or after *sample, or
 *                            (only during a leading silence longer than max_sil_kept frames: the all-silent recording's
 *                            range) lies within samples [0, *head) (head may be NULL; 0 when there is no such range); and
 *                            (rms_held, may be NULL) how many RMS values the stream holds: O(max_sil_kept).
 * The range pointers stay valid until the next call on the stream.  Concatenated over all calls, the ranges equal
 * some_slicer_ranges on the whole list (with the short-recording rule of some_session_transcribe_sliced). */
typedef struct some_slicer_stream some_slicer_stream;
int some_slicer_stream_create(const some_slicer_frames* frames, some_slicer_stream** out);
int some_slicer_stream_feed(some_slicer_stream* st, const float* rms, int n_frames, long long fixed, const int64_t** ranges,
                            int* count);
int some_slicer_stream_finish(some_slicer_stream* st, const float* rms, int n_frames, long long n_samples, const int64_t** ranges,
                              int* count);
int some_slicer_stream_keep_from(const some_slicer_stream* st, long long* sample, long long* head, long long* rms_held);
int some_slicer_stream_destroy(some_slicer_stream* st);

/* ---- Streaming (csrc/session.cu): transcribe a recording while it is still arriving.  Push samples as they come; each push
 * returns, in `out`, the chunks that became final (zero, one or several), and some_stream_finish the rest.  Concatenated in
 * order, the chunks of all pushes and the finish equal some_session_transcribe_sliced on the whole recording at the same rate
 * and params: the same [begin, end) (absolute positions at the model's rate) and bit-identical notes, however the recording is
 * split into pushes.  A chunk is delivered by the push that makes known the first voiced frame after the silent run that ends
 * it, or frame max(ss + 2 max_sil_kept, ss + min_interval - 1, chunk begin + min_length - 1) of a longer run (see
 * some_slicer_stream_feed).  With the default params at 44.1 kHz: when singing resumes after at least 300 ms of silence, or at
 * the latest about 2.1 s into a longer silence.  A frame is known once the samples it reads are fixed: at the model's rate
 * when they are received; at another rate once the resampler's right wing behind them has been received (<= 64 input samples
 * when upsampling, nwin / index_step when downsampling).
 *   Each push uploads its samples through pinned memory, resamples the outputs they fix (some_resample_kaiser_windows),
 * computes the RMS frames those complete (some_slicer_rms_windows), downloads them with one synchronise, takes the slicer's
 * decisions on the host (some_slicer_stream_*, csrc/slicer.cu) and transcribes the final chunks where they lie in the
 * stream's device buffer.  The buffer keeps only what a later chunk or RMS frame can read: `held` stays within the longest
 * chunk plus 2 max_sil_kept frames and the RMS window (during a long leading silence: the first and the last max_sil_kept
 * frames and the RMS window), plus the push in progress, however long the recording or its silences; until more than
 * min_length hops are fixed (the recording may still prove to be one chunk) it holds everything so far.
 *   Any number of streams may share a session, from different threads: pushes that queue behind a running step are run as
 * one step (see "Calls from several threads").  One stream is used by one thread at a time.  sample_rate: any integer rate (params NULL: Slicer(sr, max_sil_kept=1000)).  At finish, a
 * recording too short to resample is refused as resampy refuses it; an empty stream finishes like transcribe_sliced on zero
 * samples.  No push after finish.  Close a session's streams before the session: a stream uses its session's device, streams
 * and buffers. */
typedef struct some_stream some_stream;
typedef struct {
  int64_t received; /* samples pushed, at the stream's rate */
  int64_t fixed;    /* model-rate samples whose values can no longer change */
  int64_t held;     /* model-rate samples resident on the device */
} some_stream_info;
int some_stream_open(some_session* s, int sample_rate, const some_slicer_params* params, some_stream** out);
int some_stream_push(some_stream* st, const float* samples, long long n, some_notes* out);
int some_stream_finish(some_stream* st, some_notes* out);
int some_stream_get_info(const some_stream* st, some_stream_info* info);
int some_stream_close(some_stream* st);
/* Many streams: advances `count` streams of one session in one step.  For stream i, the effect is some_stream_push(streams[i],
 * samples[i], n[i], out[i]), followed by some_stream_finish when finish != NULL and finish[i] != 0.  out[i] receives the
 * chunks of both.  finish may be NULL.
 *   Each stream keeps the contract above, over any mix of push, finish and push_many calls, and gets each chunk in the call in
 * which some_stream_push would deliver it.  The streams of one call may have different rates and slicer params.  The call
 * does the GPU work once for all of them: one upload, one resampling and one RMS launch, one synchronise, and every chunk that
 * became final in any of the streams in one batch through the model.  So every stream of a call waits for the chunks of all.
 *   Refused, with the index i in the message and no stream changed, when: an array is NULL or count < 0; a stream is NULL,
 * belongs to another session than stream 0, appears twice or has finished; n[i] < 0, or samples[i] is NULL while n[i] > 0;
 * two entries share one some_notes; a resampling stream is to finish with too few input samples to resample.  count == 0
 * does nothing.  A failure after that (a device error) is reported like one of some_stream_push; the session stays usable,
 * but on every stream of the failed call only some_stream_get_info and some_stream_close remain defined.
 *   The call is one request (see "Calls from several threads").  Threads may call it on disjoint sets of streams of one
 * session, mixed with single pushes on other streams; one stream is used by one thread at a time. */
int some_stream_push_many(some_stream* const* streams, const float* const* samples, const long long* n, const int* finish,
                          int count, some_notes* const* out);
/* Encoded streams: a WAV, FLAC or AIFF file pushed as its bytes arrive (a recorder or encoder writing to a pipe, an upload),
 * decoded and down-mixed on the GPU exactly as some_session_transcribe_encoded decodes the whole file.  The rate comes from the
 * header.
 *   For a file that some_session_transcribe_encoded accepts, pushed in order and split in any way (single bytes, any sizes, all
 * at once), the chunks of all pushes and the finish, concatenated, equal some_session_transcribe_encoded on the whole file:
 * the same ranges and bit-identical notes.  Each chunk comes in the push where some_stream_push would deliver it if that push
 * carried the samples decoded in it: a FLAC sample is decoded once its whole frame has arrived and its CRC-16 is checked, a
 * WAV or AIFF sample once its whole sample frame has arrived.  A header whose sizes are placeholders (as recorders writing to a pipe
 * leave them) reads to the end of the bytes, as some_session_transcribe_encoded reads such a file.  One difference: a WAV file
 * with a second data chunk, or with a fmt chunk after its data chunk, is refused when that chunk's header arrives (a stream
 * cannot take back the samples of the first data chunk nor change the format they were decoded in; the whole-file call reads
 * the last of each, as scipy does).
 *   some_stream_finish, some_stream_get_info and some_stream_close serve both kinds of stream; `received` counts samples
 * decoded at the file's rate.  some_stream_push and some_stream_push_many refuse encoded streams; some_stream_push_bytes* refuse
 * PCM streams.  some_stream_get_meta: the file's metadata once the header is complete (zero before: container 0), the bytes
 * pushed and the bytes the stream holds on the host.
 *   Refusals come at the push that makes them certain, or at the finish, with the message some_session_transcribe_encoded
 * gives for the file, prefixed by the function's name (and in the many-call by "stream i"): anything some_audio_info refuses,
 * a corrupt FLAC stream (some_flac_chain's message; byte offsets from the file's first byte), a frame that fails to decode,
 * and, at the push that completes the header, a rate pair the resampler does not support, a mono down-mix of more than 128
 * channels or FLAC above 24 bits.  Chunks delivered before stay delivered; after such a refusal only some_stream_get_info,
 * some_stream_get_meta and some_stream_close remain defined on the stream, and the session stays usable.  A content refusal
 * returns SOME_STREAM_REFUSED (< 0, distinct from other errors) with the first refusal's message: in the many-call the other
 * streams have completed their step and their out[i] hold their chunks (a refused stream's out[i] holds none), so a caller
 * reads every out[i] after it, as after success.  Any other error (< 0, not SOME_STREAM_REFUSED) leaves every out[i]
 * untouched: argument errors (those of some_stream_push_many, and a PCM stream or a refused one) change no stream; after a
 * device error only some_stream_get_info, some_stream_get_meta and some_stream_close remain defined on the call's streams.
 *   Each step: the walk of each stream's bytes on the host; one pinned upload of the FLAC windows (the bytes from each stream's
 * first frame not decoded yet) and the whole WAV sample frames; with FLAC streams, one some_flac_scan, one download of the
 * candidates, one synchronise and each stream's chain (some_flac_chain_resume); then one some_pcm_decode and one FLAC decode
 * into the region some_stream_push_many's step scatters, and that step.  On top of a PCM stream's memory, an encoded stream
 * holds on the host the bytes of at most one incomplete FLAC frame or WAV sample frame, plus the push in progress, and nothing
 * of skipped metadata; on the device the session keeps the decoder scratch of one step. */
enum { SOME_STREAM_REFUSED = -3 };
int some_stream_open_encoded(some_session* s, const some_slicer_params* params, some_stream** out);
int some_stream_push_bytes(some_stream* st, const void* data, long long n_bytes, some_notes* out);
int some_stream_push_bytes_many(some_stream* const* streams, const void* const* data, const long long* n_bytes, const int* finish,
                                int count, some_notes* const* out);
int some_stream_get_meta(const some_stream* st, some_audio_meta* meta, long long* bytes_received, long long* bytes_held);
/* Provisional notes: the part of a stream the slicer has not closed yet, transcribed on demand, without waiting for the
 * chunk to be delivered.  A stream's open region is [a, b) in model-rate samples: a = the first sample of a range not returned
 * yet (some_slicer_stream_keep_from's *sample: 0 until more than min_length hops are fixed), b = `fixed` of
 * some_stream_get_info.  If b > a, `out` receives one clip with begin = a, end = b and the notes some_session_transcribe gives
 * for samples [a, b) of the recording at the model's rate (for a stream at another rate: of audio.resample of the whole input;
 * for an encoded stream: of the decoded file), bit for bit; if b == a, zero clips and no GPU work.  A peek changes nothing in
 * the stream: the chunks of all pushes and the finish are the same with or without peeks.  It works on PCM and encoded
 * streams alike; an encoded stream's samples are decoded already, so a peek decodes nothing.
 *   For each stream, a never decreases from one peek to the next, is never before the end of a chunk already delivered, and
 * every chunk delivered later begins at or after it, with one exception (some_slicer_stream_keep_from's head): a recording
 * that ends inside a leading silence longer than max_sil_kept frames is one chunk [0, e) with e <= max_sil_kept hops, which
 * begins before the a of the peeks made during that silence.
 *   Cost: the trunk runs over the whole open region at every peek, so the work grows with the region's length times the peek
 * rate; the caller chooses the rate, and the region spans the chunk in progress and any silence after it.  Each call is one step: the
 * regions of all its streams are copied, on the device, next to each other and transcribed as one batch (spread over the
 * replicas of a multi-device session like the chunks of any call), with one synchronise.
 *   some_stream_peek_many peeks `count` streams of one session in one call; out[i] receives stream i's clip.  Refused, with
 * the index i in the message and no stream or out[i] changed, when: an array is NULL or count < 0; a stream is NULL, belongs
 * to another session than stream 0, appears twice, has finished or was refused on its content; two entries share one
 * some_notes.  count == 0 does nothing.  A device error fails the call like any other; since a peek changes no stream state,
 * the session and its streams stay usable after it, and every out[i] is left untouched.
 *   Each call is one request (see "Calls from several threads"): peeks share a step with other peeks, never with a call that
 * touches the same stream or some_notes, and run after every earlier call on their streams. */
int some_stream_peek(some_stream* st, some_notes* out);
int some_stream_peek_many(some_stream* const* streams, int count, some_notes* const* out);

/* ---- Audio already on the GPU: float32 recordings in device memory (a vocal stem a separation model left there, often stereo)
 * into the session and its PCM streams, down-mixed as librosa.to_mono does, with no host copy.  An item is `channels` x
 * `frames` floats; sample (c, f) lies at data + c * channel_stride + f * frame_stride.  The layout follows from the strides
 * (some_downmix_layout): a one-dimensional recording (one channel, channel_stride 0, frame_stride 1), planar (frame_stride 1,
 * channel_stride >= frames: librosa's C-contiguous [channels, n], or a view of one with a larger channel stride) or
 * interleaved (channel_stride 1, frame_stride = channels: librosa's [channels, n] view of an [n, channels] array); any other
 * stride pattern is refused.  The mono samples are np.mean(y, axis=0) of that (channels, frames) view in float32, bit for bit,
 * in numpy's order for the layout (K-downmix).
 *   some_session_transcribe_device: for item i, out[i] receives what some_session_transcribe_sliced(s, m, frames,
 * sample_rate, params, out[i]) gives for its host down-mix m = np.mean(y, axis=0): the same chunk ranges, bit-identical notes
 * and, with some_notes_set_frames, bit-identical frame curves.  Results do not depend on the other items.  The call is one
 * recordings request (see "Calls from several threads"): it shares a step with sliced and encoded calls, counting each item's
 * model-rate samples against SOME_SESSION_STEP_SAMPLES; the step down-mixes every device item with one some_downmix launch
 * into the recording buffer, then resamples, cuts and transcribes as for host recordings.
 *   some_stream_push_device: the effect of some_stream_push of the item's down-mixed samples; sample_rate must equal the
 * stream's.  Host and device pushes may be mixed on one stream and split in any way; the chunks stay those of
 * some_session_transcribe_sliced.  The stream step down-mixes device items straight into the stream's window.
 * some_stream_push_device_many is some_stream_push_many with device items (and its refusals, encoded streams included); it
 * shares a step with any PCM push request.
 *   Ordering: at the call, an event is recorded on each item's `stream` (0: the legacy default stream of `device`), and the
 * session's stream waits on it before its first read of the item; nothing else is enqueued on the caller's streams, and the
 * caller need not synchronise.  When a call returns, the session no longer reads its items: the caller may overwrite or free
 * them.  Items may lie on any visible device; an item on another device than the session's first is copied to it
 * (cudaMemcpyPeerAsync, packed) before the down-mix; peer access is used when the application has enabled it, not required.
 *   Memory: besides what the same host call holds, the session keeps (grow-only) room for the packed copies of a step's items
 * on other devices; items on its own device are read where they lie.
 *   Refused before any GPU work, with the index i in the message and no out[i] touched: the refusals of the host calls (NULL
 * arrays, count < 0, NULL or shared some_notes, finished or encoded streams, ...); data NULL with frames > 0, or frames < 0;
 * channels outside 1..128; a stride pattern that is none of the three layouts; data that cudaPointerGetAttributes does not
 * report as device memory of `device` (a host pointer, for one); a rate pair the resampler refuses or a recording too short to
 * resample.  The session stays usable after a refusal.  count == 0 does nothing. */
typedef struct {
  const float* data;        /* device memory of `device` */
  int device;
  long long frames;
  int channels;             /* 1..128 */
  long long channel_stride; /* in floats; the layout follows from the two strides */
  long long frame_stride;
  int sample_rate;
  cudaStream_t stream;      /* the stream that produced `data` (0: legacy default stream of `device`) */
} some_device_audio;
int some_session_transcribe_device(some_session* s, const some_device_audio* items, int count, const some_slicer_params* params,
                                   some_notes* const* out);
int some_stream_push_device(some_stream* st, const some_device_audio* a, some_notes* out);
int some_stream_push_device_many(some_stream* const* streams, const some_device_audio* items, const int* finish, int count,
                                 some_notes* const* out);

#ifdef __cplusplus
}
#endif
#endif /* SOME_B200_H_ */
