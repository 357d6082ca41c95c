// K-downmix: librosa.to_mono of float32 audio already in device memory (a vocal stem a separation model left on the GPU),
// many recordings in one launch.  Output sample f of a recording is np.mean(y, axis=0) of librosa's (channels, n) view, bit for
// bit, and numpy's order depends on the memory layout (downmix.cuh):
//   mono         a one-dimensional recording: the value itself;
//   planar       frames contiguous, channel stride >= frames: the rows added in order from +0.0, then / channels
//                (mono_mean_planar);
//   interleaved  channels contiguous, frame stride = channels: numpy's pairwise sum (mono_mean), as the PCM decoder and the
//                FLAC emitter down-mix; a recording of one frame takes this order whatever its channel stride, because numpy
//                then reduces the channels as its only axis.
// Work split: each CTA writes a tile of one recording and finds its recording from the tiles' prefix sums (window_of), as
// some_pcm_decode does.  Mono and planar tiles are DM_TILE frames: thread t reads frames t + k DM_THREADS (k < DM_PER) of every
// channel, all of a channel's frames in flight together, so each channel's loads are coalesced across the warp.  An interleaved tile is the DM_STAGE / channels frames whose samples fill the stage: the
// CTA copies them, contiguous in memory, into shared memory with coalesced loads (one padding word per 32, so that the threads
// of a warp reading frames f .. f + 31 of one channel hit different banks for the common channel counts), then each thread
// reduces its frames from there.  Stores are one float per frame, consecutive across the warp.
#include <stddef.h>

#include "downmix.cuh"
#include "host_common.h"

#include "../../include/some_b200.h"

namespace some {
namespace {

constexpr int DM_THREADS = 256;
constexpr int DM_PER = 4;                 // mono and planar frames per thread
constexpr int DM_TILE = DM_PER * DM_THREADS;   // mono and planar frames per CTA
constexpr int DM_STAGE = 8192;            // interleaved samples staged per CTA (32 KB)

// The frames of one interleaved tile.
__host__ __device__ constexpr int stage_frames(int channels) { return DM_STAGE / channels; }

struct DownmixParams {
  const float* data;
  float* out;
  long long frames, cs;
  int channels, layout;
};

__global__ void __launch_bounds__(DM_THREADS) downmix_kernel(const DownmixParams* __restrict__ ps,
                                                             const long long* __restrict__ tile0, int K) {
  __shared__ float stage[DM_STAGE + DM_STAGE / 32];
  const long long tile = blockIdx.x;
  const int w = window_of(tile0, K, tile);
  const DownmixParams p = ps[w];
  const long long t = tile - __ldg(tile0 + w);
  const int ch = p.channels;
  if (p.layout == SOME_DOWNMIX_INTERLEAVED && p.frames > 1) {     // uniform over the CTA: the barrier is reached by all
    const int per = stage_frames(ch);
    const long long f0 = t * per;
    const int nf = static_cast<int>(min(static_cast<long long>(per), p.frames - f0));
    const int n = nf * ch;
    const float* __restrict__ src = p.data + f0 * ch;
#pragma unroll 8
    for (int j = threadIdx.x; j < n; j += DM_THREADS) stage[j + (j >> 5)] = __ldg(src + j);
    __syncthreads();
    for (int f = threadIdx.x; f < nf; f += DM_THREADS)
      p.out[f0 + f] = mono_mean(ch, [&](int c) {
        const int j = f * ch + c;
        return stage[j + (j >> 5)];
      });
    return;
  }
  // mono and planar: frame f0 + k DM_THREADS for k < DM_PER, every channel's loads of them in flight together
  const long long f0 = t * DM_TILE + threadIdx.x, f1 = min(p.frames, t * DM_TILE + DM_TILE);
  if (p.layout == SOME_DOWNMIX_INTERLEAVED) {                     // one frame, read at its channel stride
    if (f0 < f1) p.out[f0] = mono_mean(ch, [&](int c) { return __ldg(p.data + c * p.cs); });
    return;
  }
  float v[DM_PER];
  if (p.layout == SOME_DOWNMIX_MONO) {
#pragma unroll
    for (int k = 0; k < DM_PER; ++k) v[k] = f0 + k * DM_THREADS < f1 ? __ldg(p.data + f0 + k * DM_THREADS) : 0.f;
  } else {
    mono_mean_planar(ch, [&](int c, int k) {
      const long long f = f0 + k * DM_THREADS;
      return f < f1 ? __ldg(p.data + c * p.cs + f) : 0.f;
    }, v);
  }
#pragma unroll
  for (int k = 0; k < DM_PER; ++k)
    if (f0 + k * DM_THREADS < f1) p.out[f0 + k * DM_THREADS] = v[k];
}

}  // namespace
}  // namespace some

using namespace some;

extern "C" int some_downmix_layout(int channels, long long frames, long long channel_stride, long long frame_stride,
                                   int* layout) {
  SOME_REQUIRE(layout != nullptr, "some_downmix_layout: null pointer");
  SOME_REQUIRE(channels >= 1 && channels <= kMonoMaxChannels, "%d channels (1 to %d)", channels, kMonoMaxChannels);
  SOME_REQUIRE(frames >= 0, "%lld frames", frames);
  SOME_REQUIRE(channel_stride >= 0 && frame_stride >= 0, "negative strides (channel %lld, frame %lld)", channel_stride,
               frame_stride);
  if (channels == 1 && channel_stride == 0 && (frame_stride == 1 || frames <= 1)) {
    *layout = SOME_DOWNMIX_MONO;
  } else if (frames <= 1 && (channels == 1 || channel_stride >= 1)) {
    *layout = SOME_DOWNMIX_INTERLEAVED;         // numpy reduces the channels as the only axis: its pairwise order
  } else if (channel_stride == 1 && frame_stride == channels) {
    *layout = SOME_DOWNMIX_INTERLEAVED;
  } else if (frame_stride == 1 && (channel_stride >= frames || channels == 1)) {
    *layout = SOME_DOWNMIX_PLANAR;
  } else {
    SOME_REQUIRE(false,
                 "strides (channel %lld, frame %lld) of %d channels x %lld frames are none of the down-mix layouts: mono "
                 "(one channel, channel stride 0, frame stride 1), planar (frame stride 1, channel stride >= frames) or "
                 "interleaved (channel stride 1, frame stride = channels)",
                 channel_stride, frame_stride, channels, frames);
  }
  return 0;
}

extern "C" long long some_downmix_bytes(int K) { return K < 0 ? -1 : static_cast<long long>(windows_bytes<DownmixParams>(K)); }

extern "C" int some_downmix_pack(const some_downmix_item* items, int K, void* desc) {
  SOME_REQUIRE(desc && K >= 0 && (K == 0 || items), "some_downmix_pack: bad arguments");
  DownmixParams* ps = windows_params<DownmixParams>(desc, K);
  long long* tile0 = windows_tile0(desc);
  for (int i = 0; i < K; ++i) {
    const some_downmix_item& it = items[i];
    SOME_REQUIRE(it.channels >= 1 && it.channels <= kMonoMaxChannels && it.frames >= 0,
                 "some_downmix_pack: item %d: %lld frames of %d channels (1 to %d)", i, it.frames, it.channels,
                 kMonoMaxChannels);
    SOME_REQUIRE(it.frames == 0 || (it.data && it.out), "some_downmix_pack: item %d: null pointer", i);
    const int ly = it.layout;
    SOME_REQUIRE(ly == SOME_DOWNMIX_MONO || ly == SOME_DOWNMIX_PLANAR || ly == SOME_DOWNMIX_INTERLEAVED,
                 "some_downmix_pack: item %d: unknown layout %d", i, ly);
    SOME_REQUIRE(ly != SOME_DOWNMIX_MONO || it.channels == 1, "some_downmix_pack: item %d: mono with %d channels", i,
                 it.channels);
    SOME_REQUIRE(ly != SOME_DOWNMIX_PLANAR || it.frames <= 1 || it.channels == 1 || it.channel_stride >= it.frames,
                 "some_downmix_pack: item %d: planar channel stride %lld below %lld frames", i, it.channel_stride, it.frames);
    SOME_REQUIRE(ly == SOME_DOWNMIX_MONO || it.channels == 1 || it.channel_stride >= 1 ||
                     (ly == SOME_DOWNMIX_INTERLEAVED && it.frames > 1),
                 "some_downmix_pack: item %d: channel stride %lld", i, it.channel_stride);
    ps[i] = DownmixParams{it.data, it.out, it.frames, it.channel_stride, it.channels, ly};
    const long long per = ly == SOME_DOWNMIX_INTERLEAVED && it.frames > 1 ? stage_frames(it.channels) : DM_TILE;
    tile0[i + 1] = (it.frames + per - 1) / per;
  }
  windows_index(desc, K, 0);
  SOME_REQUIRE(windows_tile0(desc)[K] < (1ll << 31), "some_downmix_pack: grid too large");
  return 0;
}

extern "C" int some_downmix(const void* desc, const void* desc_d, cudaStream_t stream) {
  SOME_REQUIRE(desc && desc_d && reinterpret_cast<uintptr_t>(desc_d) % 16 == 0, "some_downmix: bad arguments");
  const WindowsHeader& h = *static_cast<const WindowsHeader*>(desc);
  if (h.tiles == 0) return 0;
  const int K = static_cast<int>(h.K);
  void* d = const_cast<void*>(desc_d);
  downmix_kernel<<<static_cast<unsigned>(h.tiles), DM_THREADS, 0, stream>>>(windows_params<DownmixParams>(d, K),
                                                                          windows_tile0(d), K);
  return check_launch("some_downmix");
}
