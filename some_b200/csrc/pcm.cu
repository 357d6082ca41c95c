// K-pcm: the samples of RIFF/WAVE data chunks as audio.decode_wav hands them to librosa.load (libsndfile's scaling, read
// through scipy.io.wavfile), many recordings in one launch, from their bytes on the device.
//   u8 -> (x - 128) / 128; s16 / s24 / s32 -> x / 2^(bits - 1) (s32 is rounded to float32 first, as numpy's astype does; the
//   division by a power of two is exact); f32 as is; f64 rounded to nearest float32.
// Samples may start at any byte: every sample is assembled from its bytes, so 24-bit and unaligned float samples need no
// alignment.  Mono output is np.mean's float32 order over the channels (mono_mean, downmix.cuh, shared with the FLAC
// emitter); otherwise the output is interleaved [n, channels].
// Work split: each CTA writes a fixed tile of PCM_TILE output frames of one recording and finds its recording from the tiles'
// prefix sums (window_of), as some_resample_kaiser_windows does; the descriptors travel in the caller's upload.
#include <stddef.h>

#include "downmix.cuh"
#include "host_common.h"

#include "../../include/some_b200.h"

namespace some {
namespace {

constexpr int PCM_THREADS = 256;
constexpr int PCM_TILE = 4 * PCM_THREADS;   // output frames per CTA

struct PcmParams {
  const uint8_t* data;
  float* out;
  long long frames;
  int channels, kind, mono, isz;
};

__device__ __forceinline__ float pcm_sample(const uint8_t* __restrict__ p, int kind) {
  switch (kind) {
    case SOME_PCM_U8:
      return __fmul_rn(__fsub_rn(static_cast<float>(__ldg(p)), 128.f), 0.0078125f);
    case SOME_PCM_S16: {
      const int16_t v = static_cast<int16_t>(__ldg(p) | (__ldg(p + 1) << 8));
      return __fmul_rn(static_cast<float>(v), 3.0517578125e-05f);                     // 2^-15
    }
    case SOME_PCM_S24: {                                                               // left-justified in int32, as scipy
      const int32_t v = static_cast<int32_t>((static_cast<uint32_t>(__ldg(p)) << 8) | (static_cast<uint32_t>(__ldg(p + 1)) << 16) |
                                             (static_cast<uint32_t>(__ldg(p + 2)) << 24));
      return __fmul_rn(__int2float_rn(v), 4.656612873077393e-10f);                    // 2^-31
    }
    case SOME_PCM_S32: {
      const int32_t v = static_cast<int32_t>(static_cast<uint32_t>(__ldg(p)) | (static_cast<uint32_t>(__ldg(p + 1)) << 8) |
                                             (static_cast<uint32_t>(__ldg(p + 2)) << 16) | (static_cast<uint32_t>(__ldg(p + 3)) << 24));
      return __fmul_rn(__int2float_rn(v), 4.656612873077393e-10f);
    }
    case SOME_PCM_F32: {
      const uint32_t u = static_cast<uint32_t>(__ldg(p)) | (static_cast<uint32_t>(__ldg(p + 1)) << 8) |
                         (static_cast<uint32_t>(__ldg(p + 2)) << 16) | (static_cast<uint32_t>(__ldg(p + 3)) << 24);
      return __uint_as_float(u);
    }
    default: {                                                                         // SOME_PCM_F64
      unsigned long long u = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) u |= static_cast<unsigned long long>(__ldg(p + k)) << (8 * k);
      return __double2float_rn(__longlong_as_double(static_cast<long long>(u)));
    }
  }
}

__global__ void __launch_bounds__(PCM_THREADS) pcm_decode_kernel(const PcmParams* __restrict__ ps,
                                                                 const long long* __restrict__ tile0, int K) {
  const long long tile = blockIdx.x;
  const int w = window_of(tile0, K, tile);
  const PcmParams p = ps[w];
  const long long f0 = (tile - __ldg(tile0 + w)) * PCM_TILE;
  const long long f1 = min(p.frames, f0 + PCM_TILE);
  const int ch = p.channels;
  for (long long f = f0 + threadIdx.x; f < f1; f += PCM_THREADS) {
    const uint8_t* row = p.data + f * ch * p.isz;
    if (p.mono) {
      p.out[f] = mono_mean(ch, [&](int c) { return pcm_sample(row + static_cast<long long>(c) * p.isz, p.kind); });
    } else {
      for (int c = 0; c < ch; ++c) p.out[f * ch + c] = pcm_sample(row + static_cast<long long>(c) * p.isz, p.kind);
    }
  }
}

int sample_bytes(int kind) {
  return kind == SOME_PCM_U8 ? 1 : kind == SOME_PCM_S16 ? 2 : kind == SOME_PCM_S24 ? 3 : kind == SOME_PCM_F64 ? 8
         : (kind == SOME_PCM_S32 || kind == SOME_PCM_F32) ? 4 : 0;
}

}  // namespace
}  // namespace some

using namespace some;

extern "C" long long some_pcm_decode_bytes(int K) { return K < 0 ? -1 : static_cast<long long>(windows_bytes<PcmParams>(K)); }

extern "C" int some_pcm_decode_pack(const some_pcm_item* items, int K, void* desc) {
  SOME_REQUIRE(desc && K >= 0 && (K == 0 || items), "some_pcm_decode_pack: bad arguments");
  PcmParams* ps = windows_params<PcmParams>(desc, K);
  long long* tile0 = windows_tile0(desc);
  for (int i = 0; i < K; ++i) {
    const some_pcm_item& it = items[i];
    const int isz = sample_bytes(it.kind);
    SOME_REQUIRE(isz > 0, "some_pcm_decode_pack: item %d: unknown sample kind %d", i, it.kind);
    SOME_REQUIRE(it.frames >= 0 && it.channels >= 1, "some_pcm_decode_pack: item %d: %lld frames of %d channels", i, it.frames,
                 it.channels);
    SOME_REQUIRE(!it.mono || it.channels <= kMonoMaxChannels,
                 "some_pcm_decode_pack: item %d: a mono down-mix of %d channels (numpy's order is restated up to %d)", i,
                 it.channels, kMonoMaxChannels);
    SOME_REQUIRE(it.frames == 0 || (it.data && it.out), "some_pcm_decode_pack: item %d: null pointer", i);
    ps[i] = PcmParams{it.data, it.out, it.frames, it.channels, it.kind, it.mono ? 1 : 0, isz};
    tile0[i + 1] = (it.frames + PCM_TILE - 1) / PCM_TILE;
  }
  windows_index(desc, K, 0);
  SOME_REQUIRE(windows_tile0(desc)[K] < (1ll << 31), "some_pcm_decode_pack: grid too large");
  return 0;
}

extern "C" int some_pcm_decode(const void* desc, const void* desc_d, cudaStream_t stream) {
  SOME_REQUIRE(desc && desc_d && reinterpret_cast<uintptr_t>(desc_d) % 16 == 0, "some_pcm_decode: bad arguments");
  const WindowsHeader& h = *static_cast<const WindowsHeader*>(desc);
  if (h.tiles == 0) return 0;
  const int K = static_cast<int>(h.K);
  void* d = const_cast<void*>(desc_d);
  pcm_decode_kernel<<<static_cast<unsigned>(h.tiles), PCM_THREADS, 0, stream>>>(windows_params<PcmParams>(d, K), windows_tile0(d), K);
  return check_launch("some_pcm_decode");
}
