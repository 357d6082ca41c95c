// K-decode: probabilities -> notes.  Restates utils/infer_utils.py:9-76 and the postprocess glue of
// inference/me_infer.py:78-97 / inference/me_quant_infer.py:21-38 (masks are all ones on the inference path,
// me_infer.py:62, so the mask multiplications are identities).  Three launches per call:
//
//   phase A  decode_frames_kernel, grid over ALL frames (warp per frame): argmax over the N pitch bins; continuous:
//            weighted mean of the bin values over [c-3, c+3] (infer_utils.py:11-22), rest = max < threshold (:23);
//            quantized: value = clip(argmax, 0, 127), rest = argmax == 128 (me_quant_infer.py:28-31).  This is the only
//            phase that touches the [M, N] probabilities (HBM-bound stream).
//   phase B  decode_align_kernel, one CTA per clip: boundary alignment (infer_utils.py:27-39): cumsum().round().long(),
//            diff(prepend -1) > 0, cumsum.  The float cumsum is the only order-sensitive step: ATen's CPU kernel accumulates
//            sequentially in double and rounds every prefix to float, so one thread does exactly that (a chain of T DADDs,
//            ~15 us for 30 s, all clips in parallel); everything after it is integer and runs as a block scan.
//   phase C  decode_notes_kernel, DEC_NOTE_CTAS CTAs per clip (warp per note; notes are contiguous frame ranges, so no
//            atomics on global memory): duration, unmasked duration, 128-bin histogram of round(value) -> mode (first
//            maximal bin), sequential fp32 sum of the values within +-0.5 of the mode (CPU scatter_add order), mean.
// Outputs are packed per clip at offset cu_frames[b] (a clip never has more notes than frames).
#include "host_common.h"
#include "sm90_ptx.cuh"

#include "../../include/some_b200.h"

namespace some {

constexpr int DEC_THREADS = 256;
constexpr int DEC_CHUNK = 2048;

struct DecParams {
  const float* probs;
  const float* bounds;
  const int32_t* cu_frames;
  int N;
  int quantized;
  float vmin, interval;
  int width;
  float threshold;
  float* note_midi;
  int32_t* note_dur;
  uint8_t* note_rest;
  int32_t* note_count;
  int32_t* frame2item;  // scratch or debug [M]
  float* values;        // [M]
  uint8_t* rest;        // [M]
  int32_t* note_start;  // [M]
};

constexpr int DEC_NOTE_CTAS = 16;   // CTAs per clip in phase C

// ---------------------------------------------------------------- phase A: per-frame pitch value / rest
__global__ void __launch_bounds__(DEC_THREADS) decode_frames_kernel(const DecParams p, int M) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (DEC_THREADS / 32) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int N = p.N;
  const float* __restrict__ pr = p.probs + (size_t)row * N;
  float best = -INFINITY;
  int bidx = 0x7fffffff;
  for (int j = lane; j < N; j += 32) {
    const float v = pr[j];
    if (v > best) best = v, bidx = j;  // ascending j: keeps the first maximum of this lane
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
    if (ov > best || (ov == best && oi < bidx)) best = ov, bidx = oi;
  }
  float value;
  bool is_rest;
  if (p.quantized) {
    is_rest = (bidx == 128);
    value = static_cast<float>(min(max(bidx, 0), 127));
  } else {
    const int lo = max(bidx - p.width, 0), hi = min(bidx + p.width + 1, N);
    float ps = 0.f, ws = 0.f;
    for (int j = lo; j < hi; ++j) {  // <= 7 terms, ascending (all lanes compute the same sums)
      const float w = pr[j];
      // explicit roundings (no FMA contraction): product and sums are separate fp32 ops in the reference
      ps = __fadd_rn(ps, __fmul_rn(w, __fadd_rn(__fmul_rn(static_cast<float>(j), p.interval), p.vmin)));
      ws = __fadd_rn(ws, w);
    }
    value = ps / (ws + (ws == 0.f ? 1.f : 0.f));
    is_rest = best < p.threshold;
  }
  if (lane == 0) {
    p.values[row] = value;
    p.rest[row] = is_rest ? 1 : 0;
  }
}

// ---------------------------------------------------------------- phase B: frame -> note index
__global__ void __launch_bounds__(DEC_THREADS) decode_align_kernel(const DecParams p) {
  __shared__ __align__(16) float s_f[DEC_CHUNK];
  __shared__ int s_i[DEC_CHUNK];
  __shared__ int s_warp[DEC_THREADS / 32];
  __shared__ int s_carry;
  __shared__ double s_acc;
  __shared__ int s_prev_step;

  const int clip = blockIdx.x;
  const int row0 = p.cu_frames[clip];
  const int T = p.cu_frames[clip + 1] - row0;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (T <= 0) {
    if (tid == 0) p.note_count[clip] = 0;
    return;
  }
  if (tid == 0) {
    s_acc = 0.0;
    s_prev_step = -1;
    s_carry = 0;
  }
  __syncthreads();
  for (int c0 = 0; c0 < T; c0 += DEC_CHUNK) {
    const int n = min(DEC_CHUNK, T - c0);
    for (int i = tid; i < n; i += DEC_THREADS) s_f[i] = p.bounds[row0 + c0 + i];
    __syncthreads();
    if (tid == 0) {
      double acc = s_acc;
      int i = 0;
      // the DADD chain is the critical path; loads / conversions / stores of four frames are batched around it
      for (; i + 4 <= n; i += 4) {
        const float4 v = *reinterpret_cast<const float4*>(&s_f[i]);
        float4 o;
        acc += static_cast<double>(v.x), o.x = static_cast<float>(acc);  // prefix rounded to float, like ATen's CPU cumsum
        acc += static_cast<double>(v.y), o.y = static_cast<float>(acc);
        acc += static_cast<double>(v.z), o.z = static_cast<float>(acc);
        acc += static_cast<double>(v.w), o.w = static_cast<float>(acc);
        *reinterpret_cast<float4*>(&s_f[i]) = o;
      }
      for (; i < n; ++i) {
        acc += static_cast<double>(s_f[i]);
        s_f[i] = static_cast<float>(acc);
      }
      s_acc = acc;
    }
    __syncthreads();
    // step = round-half-even(prefix); inc = step - previous step > 0
    for (int i = tid; i < n; i += DEC_THREADS) s_i[i] = static_cast<int>(rintf(s_f[i]));
    __syncthreads();
    const int prev0 = s_prev_step;
    // block scan of inc over the chunk: each thread owns DEC_CHUNK / DEC_THREADS consecutive frames
    constexpr int PER = DEC_CHUNK / DEC_THREADS;
    int inc[PER];
    int local = 0;
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int i = tid * PER + k;
      int v = 0;
      if (i < n) {
        const int prev = (i == 0) ? prev0 : s_i[i - 1];
        v = (s_i[i] - prev) > 0 ? 1 : 0;
      }
      inc[k] = v;
      local += v;
    }
    int incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int warp_off = 0;
    for (int w = 0; w < warp; ++w) warp_off += s_warp[w];
    int running = s_carry + warp_off + incl - local;
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int i = tid * PER + k;
      if (i < n) {
        running += inc[k];
        p.frame2item[row0 + c0 + i] = running;
        if (inc[k]) p.note_start[row0 + running - 1] = c0 + i;
      }
    }
    __syncthreads();
    if (tid == DEC_THREADS - 1) {
      s_carry = running;  // last thread's running total = notes so far (threads past n add nothing)
      s_prev_step = s_i[n - 1];
    }
    __syncthreads();
  }
  if (tid == 0) p.note_count[clip] = s_carry;
}

// ---------------------------------------------------------------- phase C: per-note reduction
__global__ void __launch_bounds__(DEC_THREADS) decode_notes_kernel(const DecParams p) {
  __shared__ int s_hist[DEC_THREADS / 32][128];
  const int clip = blockIdx.y;
  const int row0 = p.cu_frames[clip];
  const int T = p.cu_frames[clip + 1] - row0;
  if (T <= 0) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = DEC_THREADS / 32;
  const int num_notes = p.note_count[clip];
  for (int nt = blockIdx.x * NW + warp; nt < num_notes; nt += gridDim.x * NW) {
    const int start = p.note_start[row0 + nt];
    const int end = (nt + 1 < num_notes) ? p.note_start[row0 + nt + 1] : T;
    const int dur = end - start;
    for (int b = lane; b < 128; b += 32) s_hist[warp][b] = 0;
    __syncwarp();
    int unmasked = 0;
    for (int f = start + lane; f < end; f += 32) {
      if (!p.rest[row0 + f]) {
        ++unmasked;
        int b = static_cast<int>(rintf(p.values[row0 + f]));
        b = min(max(b, 0), 127);
        atomicAdd(&s_hist[warp][b], 1);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) unmasked += __shfl_xor_sync(0xffffffffu, unmasked, o);
    __syncwarp();
    int best = -1, bidx = 0x7fffffff;
    for (int b = lane; b < 128; b += 32) {
      const int h = s_hist[warp][b];
      if (h > best) best = h, bidx = b;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
      if (ov > best || (ov == best && oi < bidx)) best = ov, bidx = oi;
    }
    __syncwarp();
    if (lane == 0) {
      const float center = static_cast<float>(bidx);
      float sum = 0.f;
      int valid = 0;
      for (int f = start; f < end; ++f) {  // frame order, fp32: the CPU scatter_add order
        const float v = p.values[row0 + f];
        if (!p.rest[row0 + f] && v >= center - 0.5f && v <= center + 0.5f) {
          sum = __fadd_rn(sum, v);
          ++valid;
        }
      }
      p.note_midi[row0 + nt] = sum / static_cast<float>(valid + (valid == 0 ? 1 : 0));
      p.note_dur[row0 + nt] = dur;
      const bool item_mask = (static_cast<float>(unmasked) / static_cast<float>(dur)) >= 0.5f;
      p.note_rest[row0 + nt] = item_mask ? 0 : 1;
    }
    __syncwarp();
  }
}

}  // namespace some

using namespace some;

extern "C" uint64_t some_decode_scratch_bytes(int M) { return 16ull * (M > 0 ? M : 0) + 256; }

extern "C" int some_decode_notes(const some_decode_args* a, cudaStream_t stream) {
  SOME_REQUIRE(a != nullptr, "some_decode_notes: null args");
  if (a->B <= 0) return 0;
  SOME_REQUIRE(a->probs && a->bounds && a->cu_frames && a->note_midi && a->note_dur && a->note_rest && a->note_count &&
                   a->scratch,
               "some_decode_notes: null pointer");
  SOME_REQUIRE(a->N >= 2 && a->N <= 256, "some_decode_notes: N=%d out of range", a->N);
  if (a->quantized) SOME_REQUIRE(a->N == 129, "some_decode_notes: quantized decode expects 129 bins (rest = 128)");
  DecParams p;
  p.probs = a->probs, p.bounds = a->bounds, p.cu_frames = a->cu_frames;
  p.N = a->N, p.quantized = a->quantized;
  p.vmin = a->vmin;
  // infer_utils.py:11-12 (python floats): interval = (vmax - vmin) / (N - 1); width = int(3 * deviation / interval)
  const double interval = (static_cast<double>(a->vmax) - static_cast<double>(a->vmin)) / (a->N - 1);
  p.interval = static_cast<float>(interval);
  p.width = a->quantized ? 0 : static_cast<int>(3.0 * static_cast<double>(a->deviation) / interval);
  p.threshold = a->threshold;
  p.note_midi = a->note_midi, p.note_dur = a->note_dur, p.note_rest = a->note_rest, p.note_count = a->note_count;
  uint8_t* s = static_cast<uint8_t*>(a->scratch);
  const size_t M = static_cast<size_t>(a->M);
  p.frame2item = a->dbg_frame2item ? a->dbg_frame2item : reinterpret_cast<int32_t*>(s);
  p.values = a->dbg_values ? a->dbg_values : reinterpret_cast<float*>(s + 4 * M);
  p.note_start = reinterpret_cast<int32_t*>(s + 8 * M);
  p.rest = a->dbg_rest ? a->dbg_rest : (s + 12 * M);
  SOME_REQUIRE(a->M > 0, "some_decode_notes: M must be positive (got %d)", a->M);
  decode_frames_kernel<<<(a->M + DEC_THREADS / 32 - 1) / (DEC_THREADS / 32), DEC_THREADS, 0, stream>>>(p, a->M);
  decode_align_kernel<<<a->B, DEC_THREADS, 0, stream>>>(p);
  decode_notes_kernel<<<dim3(DEC_NOTE_CTAS, a->B), DEC_THREADS, 0, stream>>>(p);
  return check_launch("some_decode_notes");
}
