// K-eval: validation losses and MIDI accuracy of the training tasks for labelled clips (training/me_task.py:72-154,
// training/me_quant_task.py:43-120), from the raw logits the trunk writes with the SOME_EPI_BIAS_F32 head.
//
// One CTA per clip.  Warp w takes frames w, w + 8, ... of its clip (warp per frame, the row in registers, lane l owning
// columns l + 32 k); per frame it forms the task's target on the fly (the gaussian blur of the collater, or the note's
// class), the loss terms, the activated head and the validation step's decode of it, and adds the frame's loss to a
// per-warp double.  The warps' partial sums are combined in warp order, and the bound loss (a prefix scan) is one
// sequential chain per clip over staged chunks, so every result is a fixed-order reduction that depends on its clip only.
//
// The activation must be exactly what the forward would have produced with the sigmoid / softmax head, because the
// accuracy counts and the predicted notes have to equal infer()'s (SOME_EVAL_HEAD_TC, the GEMM epilogues of gemm.cu) or
// infer_accurate()'s (SOME_EVAL_HEAD_F32, head_f32_kernel of accurate.cu):
//   sigmoid  1 / (1 + __expf(-x)) resp. 1 / (1 + expf(-x)), element-wise;
//   softmax  TC: the epilogue's quad of lanes q = 0..3 each sums __expf(x - max) over columns 8 j + 2 q + e (j ascending,
//            e inner), then two xor-shuffles (1, 2), scale by 1 / sum; F32: lane l sums expf(x - max) over l + 32 k, a
//            16..1 butterfly, divide by the sum.  The TC order is replayed from the row staged in shared memory.
#include "host_common.h"

#include <math.h>

#include "../../include/some_b200.h"

namespace some {

constexpr int EV_THREADS = 256;
constexpr int EV_WARPS = EV_THREADS / 32;
constexpr int EV_KMAX = 8;          // N <= 256 columns: 8 per lane
constexpr int EV_CHUNK = 2048;      // bound-loss staging

struct EvalParams {
  some_eval_args a;
  float interval, inv_sigma;        // me_task.py:20-21 (python floats, used as float32 scalars)
  int width;                        // infer_utils.py:12
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <bool QUANT, bool TC>
__global__ void __launch_bounds__(EV_THREADS) eval_clips_kernel(const EvalParams P) {
  __shared__ float s_row[EV_WARPS][256];
  __shared__ double s_wsum[EV_WARPS];
  __shared__ int s_wcorrect[EV_WARPS], s_wbad[EV_WARPS];
  __shared__ float s_b[EV_CHUNK];
  __shared__ int s_u[EV_CHUNK];

  const some_eval_args& a = P.a;
  const int clip = blockIdx.x;
  const int row0 = a.cu_frames[clip];
  const int T = a.cu_frames[clip + 1] - row0;
  const int note0 = a.cu_notes[clip];
  const int num_notes = a.cu_notes[clip + 1] - note0;
  const int N = a.N;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float* row_s = s_row[warp];

  double wsum = 0.0;
  int wcorrect = 0, wbad = 0;
  for (int f = warp; f < T; f += EV_WARPS) {
    const size_t r = static_cast<size_t>(row0 + f);
    const float* __restrict__ xr = a.logits + r * N;
    float x[EV_KMAX];
#pragma unroll
    for (int k = 0; k < EV_KMAX; ++k) {
      const int j = lane + 32 * k;
      x[k] = j < N ? xr[j] : -INFINITY;
    }
    const int u = a.unit2note[r];
    const bool bad = u < 1 || u > num_notes;
    wbad |= bad ? 1 : 0;
    const int note = note0 + (bad ? 0 : u - 1);
    const float nm = num_notes > 0 ? a.note_midi[note] : 0.f;
    const bool rest_gt = QUANT ? (nm == 128.f) : (num_notes > 0 && a.note_rest[note] != 0);

    // ---- loss term of the frame
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < EV_KMAX; ++k) mx = fmaxf(mx, x[k]);
    mx = warp_max(mx);
    float frame_loss;
    if constexpr (QUANT) {
      // CrossEntropyLoss: logsumexp(x) - x[target]   (stable log-softmax)
      float s = 0.f, xt = 0.f;
      const int target = static_cast<int>(nm);
#pragma unroll
      for (int k = 0; k < EV_KMAX; ++k) {
        const int j = lane + 32 * k;
        if (j < N) s += expf(x[k] - mx);
        if (j == target) xt = x[k];
      }
      s = warp_sum(s);
      xt = warp_sum(xt);        // one lane holds it, the others add +0
      frame_loss = (mx + logf(s)) - xt;
    } else {
      // BCEWithLogitsLoss against exp(-((bin - midi_to_bin(note)) / sigma)^2 / 2), zero on rests
      const float miu = (nm - a.vmin) / P.interval;
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < EV_KMAX; ++k) {
        const int j = lane + 32 * k;
        if (j < N) {
          const float t = (static_cast<float>(j) - miu) * P.inv_sigma;
          const float y = rest_gt ? 0.f : expf(__fmul_rn(t, t) / -2.0f);
          s += (fmaxf(x[k], 0.f) - x[k] * y) + log1pf(expf(-fabsf(x[k])));
        }
      }
      frame_loss = warp_sum(s);
    }
    wsum += static_cast<double>(frame_loss);

    // ---- activated head, exactly as the forward's head writes it
    float p[EV_KMAX];
    if constexpr (QUANT) {
      if constexpr (TC) {
#pragma unroll
        for (int k = 0; k < EV_KMAX; ++k) {
          const int j = lane + 32 * k;
          p[k] = j < N ? __expf(x[k] - mx) : 0.f;
          if (j < 256) row_s[j] = p[k];
        }
        __syncwarp();
        const int q = lane & 3;     // every quad replays the epilogue's quad; all lanes end with the same sum
        float sum = 0.f;
        for (int j = 0; j < 32; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * j + 2 * q + e;
            if (col < N) sum += row_s[col];
          }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum = sum + __shfl_xor_sync(0xffffffffu, sum, 2);
        const float inv = 1.0f / sum;
#pragma unroll
        for (int k = 0; k < EV_KMAX; ++k) p[k] = p[k] * inv;
        __syncwarp();
      } else {
        float sum = 0.f;
#pragma unroll
        for (int k = 0; k < EV_KMAX; ++k)
          if (lane + 32 * k < N) sum += expf(x[k] - mx);
        sum = warp_sum(sum);
#pragma unroll
        for (int k = 0; k < EV_KMAX; ++k) p[k] = lane + 32 * k < N ? expf(x[k] - mx) / sum : 0.f;
      }
    } else {
#pragma unroll
      for (int k = 0; k < EV_KMAX; ++k) {
        if constexpr (TC) p[k] = 1.0f / (1.0f + __expf(-x[k]));
        else p[k] = 1.0f / (1.0f + expf(-x[k]));
      }
    }
    if (a.probs != nullptr) {
      float* pr = a.probs + r * N;   // may alias the logits: this warp has read the whole row
#pragma unroll
      for (int k = 0; k < EV_KMAX; ++k)
        if (lane + 32 * k < N) pr[lane + 32 * k] = p[k];
    }

    // ---- the validation step's decode of the frame (same arithmetic as decode_frames_kernel) and MIDIAccuracy
    float best = -INFINITY;
    int bidx = 0x7fffffff;
#pragma unroll
    for (int k = 0; k < EV_KMAX; ++k)
      if (lane + 32 * k < N && p[k] > best) best = p[k], bidx = lane + 32 * k;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      if (ov > best || (ov == best && oi < bidx)) best = ov, bidx = oi;
    }
    bool hit;
    if constexpr (QUANT) {
      hit = bidx != 128 && !rest_gt && fabsf(static_cast<float>(bidx) - nm) <= 0.5f;
    } else {
#pragma unroll
      for (int k = 0; k < EV_KMAX; ++k)
        if (lane + 32 * k < N) row_s[lane + 32 * k] = p[k];
      __syncwarp();
      const int lo = max(bidx - P.width, 0), hi = min(bidx + P.width + 1, N);
      float ps = 0.f, ws = 0.f;
      for (int j = lo; j < hi; ++j) {
        const float w = row_s[j];
        ps = __fadd_rn(ps, __fmul_rn(w, __fadd_rn(__fmul_rn(static_cast<float>(j), P.interval), a.vmin)));
        ws = __fadd_rn(ws, w);
      }
      const float value = ps / (ws + (ws == 0.f ? 1.f : 0.f));
      const bool rest_pred = best < a.threshold;
      hit = !rest_pred && !rest_gt && fabsf(value - nm) <= 0.5f;
      __syncwarp();
    }
    wcorrect += hit ? 1 : 0;
  }
  if (lane == 0) {
    s_wsum[warp] = wsum;
    s_wcorrect[warp] = wcorrect;
    s_wbad[warp] = wbad;
  }

  // ---- BinaryEMDLoss: one sequential chain per clip (the float prefix of ATen's CPU cumsum)
  const float scale = static_cast<float>(sqrt(static_cast<double>(T)));
  double acc = 0.0, l1 = 0.0;
  int gt = 0, prev_u = 0;
  for (int c0 = 0; c0 < T; c0 += EV_CHUNK) {
    const int n = min(EV_CHUNK, T - c0);
    __syncthreads();
    for (int i = tid; i < n; i += EV_THREADS) {
      s_b[i] = a.bounds[row0 + c0 + i];
      s_u[i] = a.unit2note[row0 + c0 + i];
    }
    __syncthreads();
    if (tid == 0) {
      for (int i = 0; i < n; ++i) {
        acc += static_cast<double>(s_b[i]);
        gt += s_u[i] - prev_u > 0 ? 1 : 0;
        prev_u = s_u[i];
        const float d = static_cast<float>(acc) / scale - static_cast<float>(gt) / scale;
        l1 += static_cast<double>(fabsf(d));
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    double msum = 0.0;
    int correct = 0, bad = 0;
    for (int w = 0; w < EV_WARPS; ++w) msum += s_wsum[w], correct += s_wcorrect[w], bad |= s_wbad[w];
    a.midi_loss[clip] = bad ? NAN : msum;
    a.bound_loss[clip] = bad ? NAN : l1;
    a.correct[clip] = bad ? -1 : correct;
  }
}

}  // namespace some

using namespace some;

extern "C" int some_eval_clips(const some_eval_args* a, cudaStream_t stream) {
  SOME_REQUIRE(a != nullptr, "some_eval_clips: null args");
  if (a->B <= 0) return 0;
  SOME_REQUIRE(a->logits && a->bounds && a->cu_frames && a->unit2note && a->cu_notes && a->note_midi && a->midi_loss &&
                   a->bound_loss && a->correct,
               "some_eval_clips: null pointer");
  SOME_REQUIRE(a->quantized || a->note_rest, "some_eval_clips: the continuous task needs note_rest");
  SOME_REQUIRE(a->N >= 2 && a->N <= 256, "some_eval_clips: N=%d out of range", a->N);
  if (a->quantized) SOME_REQUIRE(a->N == 129, "some_eval_clips: the quantized task expects 129 classes (rest = 128)");
  SOME_REQUIRE(a->head == SOME_EVAL_HEAD_TC || a->head == SOME_EVAL_HEAD_F32, "some_eval_clips: bad head %d", a->head);
  SOME_REQUIRE(a->M >= 0, "some_eval_clips: bad M=%d", a->M);
  EvalParams P;
  P.a = *a;
  const double interval = (static_cast<double>(a->vmax) - static_cast<double>(a->vmin)) / (a->N - 1);
  P.interval = static_cast<float>(interval);
  P.inv_sigma = static_cast<float>(interval / static_cast<double>(a->deviation));
  P.width = a->quantized ? 0 : static_cast<int>(3.0 * static_cast<double>(a->deviation) / interval);
  const bool tc = a->head == SOME_EVAL_HEAD_TC;
  if (a->quantized)
    (tc ? eval_clips_kernel<true, true> : eval_clips_kernel<true, false>)<<<a->B, EV_THREADS, 0, stream>>>(P);
  else
    (tc ? eval_clips_kernel<false, true> : eval_clips_kernel<false, false>)<<<a->B, EV_THREADS, 0, stream>>>(P);
  return check_launch("some_eval_clips");
}
