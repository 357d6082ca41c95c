// K-rms: short-time RMS of a device-resident waveform for the silence slicer (utils/slicer2.py:5-38 `get_rms`, called from
// Slicer.slice :81 with frame_length = win_size, hop_length = hop_size, constant (zero) padding of frame_length / 2).
//
// The slicer compares every RMS value with a threshold and takes argmins over RMS windows (slicer2.py:84-133), so chunk
// boundaries are only reproducible if the RMS values are BIT-identical to numpy's.  numpy reduces the squared window along
// its contiguous axis with pairwise summation (float32): blocks of <= 128 elements are summed with 8 interleaved
// accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) plus a sequential tail, larger ranges are split at
// n/2 rounded down to a multiple of 8.  This kernel evaluates exactly that tree per frame (one thread per frame, no FMA
// contraction: __fmul_rn / __fadd_rn / __fdiv_rn / __fsqrt_rn), so the host state machine sees the same numbers as the
// reference.  13.2 M samples (5 min) -> 15 001 frames x 3528 samples: ~53 M multiply-adds, L1 / L2 resident.
#include "host_common.h"

#include <algorithm>

#include "../../include/some_b200.h"

namespace some {

struct RmsWindow {
  const float* wave;  // wave[s - base] is sample s
  long long base;
  long long n_samples;
  long long first;  // sample index of window element 0 (may be negative: zero padding)
  __device__ __forceinline__ float sq(int k) const {
    const long long s = first + k;
    const float v = (s >= 0 && s < n_samples) ? __ldg(wave + (s - base)) : 0.f;
    return __fmul_rn(v, v);
  }
};

// numpy's pairwise_sum for one block of 8 <= n <= 128 elements starting at window element lo
__device__ __forceinline__ float rms_block(const RmsWindow& w, int lo, int n) {
  float r0 = w.sq(lo), r1 = w.sq(lo + 1), r2 = w.sq(lo + 2), r3 = w.sq(lo + 3);
  float r4 = w.sq(lo + 4), r5 = w.sq(lo + 5), r6 = w.sq(lo + 6), r7 = w.sq(lo + 7);
  int i = 8;
  const int n8 = n - (n % 8);
  for (; i < n8; i += 8) {
    r0 = __fadd_rn(r0, w.sq(lo + i));
    r1 = __fadd_rn(r1, w.sq(lo + i + 1));
    r2 = __fadd_rn(r2, w.sq(lo + i + 2));
    r3 = __fadd_rn(r3, w.sq(lo + i + 3));
    r4 = __fadd_rn(r4, w.sq(lo + i + 4));
    r5 = __fadd_rn(r5, w.sq(lo + i + 5));
    r6 = __fadd_rn(r6, w.sq(lo + i + 6));
    r7 = __fadd_rn(r7, w.sq(lo + i + 7));
  }
  float res = __fadd_rn(__fadd_rn(__fadd_rn(r0, r1), __fadd_rn(r2, r3)), __fadd_rn(__fadd_rn(r4, r5), __fadd_rn(r6, r7)));
  for (; i < n; ++i) res = __fadd_rn(res, w.sq(lo + i));
  return res;
}

constexpr int RMS_MAX_DEPTH = 24;  // frame_length < 128 * 2^24

// Frames [f_begin, f_begin + n_frames) into rms[0, n_frames): a frame's value depends on its absolute index and the samples
// alone, so a window of frames over a buffer holding part of the recording gives the whole-recording bits.
__global__ void __launch_bounds__(128) slicer_rms_kernel(const float* __restrict__ wave, long long base, long long n_samples,
                                                         int frame_length, int hop, float* __restrict__ rms, long long f_begin,
                                                         int n_frames) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_frames) return;
  const long long f = f_begin + i;
  RmsWindow w{wave, base, n_samples, f * hop - frame_length / 2};
  float total;
  if (frame_length < 8) {
    total = w.sq(0);
    for (int i = 1; i < frame_length; ++i) total = __fadd_rn(total, w.sq(i));
  } else {
    // depth-first walk of numpy's split tree with an explicit stack: left subtree first, then right, then the add
    int lo_s[RMS_MAX_DEPTH], n_s[RMS_MAX_DEPTH];
    float left_s[RMS_MAX_DEPTH];
    signed char state_s[RMS_MAX_DEPTH];  // 0 = descend left, 1 = left done -> descend right, 2 = both done
    int sp = 0;
    lo_s[0] = 0, n_s[0] = frame_length, state_s[0] = 0;
    float ret = 0.f;
    while (sp >= 0) {
      const int lo = lo_s[sp], n = n_s[sp];
      if (n <= 128) {
        ret = rms_block(w, lo, n);
        --sp;
        continue;
      }
      int n2 = n / 2;
      n2 -= n2 % 8;
      if (state_s[sp] == 0) {
        state_s[sp] = 1;
        ++sp;
        lo_s[sp] = lo, n_s[sp] = n2, state_s[sp] = 0;
      } else if (state_s[sp] == 1) {
        left_s[sp] = ret;
        state_s[sp] = 2;
        ++sp;
        lo_s[sp] = lo + n2, n_s[sp] = n - n2, state_s[sp] = 0;
      } else {
        ret = __fadd_rn(left_s[sp], ret);
        --sp;
      }
    }
    total = ret;
  }
  rms[i] = __fsqrt_rn(__fdiv_rn(total, static_cast<float>(frame_length)));
}

}  // namespace some

using namespace some;

extern "C" int some_slicer_rms(const float* wave, long long n_samples, int frame_length, int hop, float* rms, int n_frames,
                               cudaStream_t stream) {
  SOME_REQUIRE(wave && rms, "some_slicer_rms: null pointer");
  SOME_REQUIRE(n_samples >= 0 && frame_length >= 1 && hop >= 1 && n_frames >= 0, "some_slicer_rms: bad sizes");
  // numpy frames the padded signal: n_frames = 1 + (n_samples + 2 * (frame_length / 2) - frame_length) / hop
  const long long padded = n_samples + 2ll * (frame_length / 2);
  SOME_REQUIRE(padded >= frame_length && n_frames == 1 + (padded - frame_length) / hop,
               "some_slicer_rms: n_frames %d does not match %lld samples, window %d, hop %d", n_frames, n_samples, frame_length, hop);
  if (n_frames == 0) return 0;
  slicer_rms_kernel<<<(n_frames + 127) / 128, 128, 0, stream>>>(wave, 0, n_samples, frame_length, hop, rms, 0, n_frames);
  return check_launch("some_slicer_rms");
}

extern "C" int some_slicer_rms_window(const float* wave, long long base, long long held, long long n_samples, int frame_length,
                                      int hop, float* rms, long long f_begin, long long f_end, cudaStream_t stream) {
  SOME_REQUIRE(wave && rms, "some_slicer_rms_window: null pointer");
  SOME_REQUIRE(base >= 0 && held >= 0 && n_samples >= -1 && frame_length >= 1 && hop >= 1 && f_begin >= 0 && f_end >= f_begin &&
                   f_end - f_begin < (1ll << 31),
               "some_slicer_rms_window: bad sizes");
  if (f_end == f_begin) return 0;
  const long long half = frame_length / 2;
  const bool final = n_samples >= 0;
  if (final) {
    const long long padded = n_samples + 2 * half;
    SOME_REQUIRE(padded >= frame_length && f_end <= 1 + (padded - frame_length) / hop,
                 "some_slicer_rms_window: frame %lld is past the last frame of %lld samples", f_end - 1, n_samples);
  }
  // the samples the frames read that lie inside the recording: the buffer must hold them
  const long long lo = std::max(0ll, f_begin * hop - half);
  const long long hi = (f_end - 1) * hop - half + frame_length;
  const long long hi_in = final ? std::min(hi, n_samples) : hi;
  SOME_REQUIRE(lo >= base && hi_in <= base + held,
               "some_slicer_rms_window: frames [%lld, %lld) read samples [%lld, %lld), the buffer holds [%lld, %lld)%s", f_begin,
               f_end, lo, hi_in, base, base + held, final ? "" : " (the recording's length is not known yet)");
  slicer_rms_kernel<<<static_cast<unsigned>((f_end - f_begin + 127) / 128), 128, 0, stream>>>(
      wave, base, final ? n_samples : base + held, frame_length, hop, rms, f_begin, static_cast<int>(f_end - f_begin));
  return check_launch("some_slicer_rms_window");
}
