// The down-mix of librosa.to_mono, shared by the FLAC emitter (flac.cu), the PCM decoder (pcm.cu) and the float32 down-mix of
// audio already on the device (downmix.cu).
#pragma once

namespace some {

// Largest channel count mono_mean restates: numpy splits longer sums recursively, which is not restated here.
constexpr int kMonoMaxChannels = 128;

// np.mean(y, axis=0) in float32 for librosa's (channels, n) view of an [n, channels] array: numpy reduces the contiguous
// channels with its pairwise sum, which is a plain left-to-right sum below 8 values and, from 8 to 128, eight running sums
// (r[j] += x[i + j]) combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), followed by the values that do not fill a
// group of eight; the sum starts from the reduction's identity +0.0 (so an all -0.0 frame gives +0.0), and is divided by the
// channel count.  One channel: the value itself (to_mono leaves a one-dimensional recording alone).  value(c) returns channel c
// of the frame as float32.  1 <= ch <= kMonoMaxChannels.
template <class F>
__device__ __forceinline__ float mono_mean(int ch, F value) {
  if (ch == 1) return value(0);
  float sum;
  if (ch < 8) {
    sum = value(0);
    for (int c = 1; c < ch; ++c) sum = __fadd_rn(sum, value(c));
  } else {
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = value(j);
    int i = 8;
    for (const int full = ch - ch % 8; i < full; i += 8)
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], value(i + j));
    sum = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])), __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < ch; ++i) sum = __fadd_rn(sum, value(i));
  }
  return __fdiv_rn(__fadd_rn(0.f, sum), static_cast<float>(ch));
}

// np.mean(y, axis=0) in float32 for a (channels, n) array whose frames are contiguous (a C-contiguous [channels, n] array,
// or a view of one with a larger channel stride), n >= 2: numpy adds the rows one after another into an output that starts
// from the identity +0.0 (so an all -0.0 frame gives +0.0, also for one channel), then divides by the channel count.  The
// order differs from mono_mean's from 8 channels up.  N frames at once, so that their loads are in flight together:
// value(c, k) returns channel c of frame k, mean[k] receives frame k's mean.  1 <= ch.
template <int N, class F>
__device__ __forceinline__ void mono_mean_planar(int ch, F value, float (&mean)[N]) {
  float sum[N];
#pragma unroll
  for (int k = 0; k < N; ++k) sum[k] = 0.f;
#pragma unroll 2
  for (int c = 0; c < ch; ++c)
#pragma unroll
    for (int k = 0; k < N; ++k) sum[k] = __fadd_rn(sum[k], value(c, k));
#pragma unroll
  for (int k = 0; k < N; ++k) mean[k] = __fdiv_rn(sum[k], static_cast<float>(ch));
}

}  // namespace some
