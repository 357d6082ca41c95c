// K-pcm: the samples of RIFF/WAVE data chunks and AIFF / AIFF-C SSND chunks as libsndfile hands them to librosa.load (for
// WAV read through scipy.io.wavfile, as audio.decode_wav does), many recordings in one launch, from their bytes on the device.
//   u8 -> (x - 128) / 128; s8 / s16 / s24 / s32, little- or big-endian -> x / 2^(8 bytes - 1) (s32 is rounded to float32
//   first, as numpy's astype does; the division by a power of two is exact); f32 as is; f64 rounded to nearest float32;
//   G.711 u-law / A-law -> libsndfile's 16-bit expansion / 32768, computed with the standard bit arithmetic (a table in
//   constant memory would serialise the lanes' different indices).
// Samples may start at any byte: every sample is assembled from its bytes, so 24-bit and unaligned float samples need no
// alignment.  Mono output is np.mean's float32 order over the channels (mono_mean, downmix.cuh, shared with the FLAC
// emitter); otherwise the output is interleaved [n, channels].
// Work split: each CTA writes a fixed tile of PCM_TILE output frames of one recording and finds its recording from the tiles'
// prefix sums (window_of), as some_resample_kaiser_windows does; the descriptors travel in the caller's upload.  The kind is
// the same for every lane of a recording, so the switch in pcm_sample does not diverge.
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
  int channels, kind, mono, isz, be;   // be: the samples are big-endian
};

// G.711 expansions to 16-bit values (ITU-T G.711; the bit arithmetic of Sun's g711.c, whose values libsndfile tabulates).
__device__ __forceinline__ int ulaw_value(uint32_t code) {
  const uint32_t u = ~code & 0xFF;
  const int t = static_cast<int>(((u & 0x0F) << 3) + 0x84) << ((u >> 4) & 7);
  return (u & 0x80) ? 0x84 - t : t - 0x84;
}
__device__ __forceinline__ int alaw_value(uint32_t code) {
  const uint32_t a = code ^ 0x55;
  const int seg = (a >> 4) & 7, m = static_cast<int>(a & 0x0F) << 4;
  const int t = seg == 0 ? m + 8 : (m + 0x108) << (seg - 1);
  return (a & 0x80) ? t : -t;
}

// One sample: its isz bytes at p as an unsigned integer in the kind's byte order (be: big-endian), then the kind's value.
__device__ __forceinline__ float pcm_sample(const uint8_t* __restrict__ p, int kind, int isz, bool be) {
  unsigned long long u = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (i < isz) u |= static_cast<unsigned long long>(__ldg(p + i)) << (8 * (be ? isz - 1 - i : i));
  const uint32_t w = static_cast<uint32_t>(u);
  switch (kind) {
    case SOME_PCM_U8:
      return __fmul_rn(__fsub_rn(static_cast<float>(w), 128.f), 0.0078125f);
    case SOME_PCM_S8:
      return __fmul_rn(static_cast<float>(static_cast<int8_t>(w)), 0.0078125f);          // 2^-7
    case SOME_PCM_S16:
    case SOME_PCM_S16BE:
      return __fmul_rn(static_cast<float>(static_cast<int16_t>(w)), 3.0517578125e-05f);  // 2^-15
    case SOME_PCM_S24:                                                                 // left-justified in int32, as scipy
    case SOME_PCM_S24BE:
      return __fmul_rn(__int2float_rn(static_cast<int32_t>(w << 8)), 4.656612873077393e-10f);   // 2^-31
    case SOME_PCM_S32:
    case SOME_PCM_S32BE:
      return __fmul_rn(__int2float_rn(static_cast<int32_t>(w)), 4.656612873077393e-10f);
    case SOME_PCM_F32:
    case SOME_PCM_F32BE:
      return __uint_as_float(w);
    case SOME_PCM_ULAW:
      return __fmul_rn(static_cast<float>(ulaw_value(w)), 3.0517578125e-05f);
    case SOME_PCM_ALAW:
      return __fmul_rn(static_cast<float>(alaw_value(w)), 3.0517578125e-05f);
    default:                                                                           // SOME_PCM_F64, SOME_PCM_F64BE
      return __double2float_rn(__longlong_as_double(static_cast<long long>(u)));
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
      p.out[f] = mono_mean(ch, [&](int c) { return pcm_sample(row + static_cast<long long>(c) * p.isz, p.kind, p.isz, p.be); });
    } else {
      for (int c = 0; c < ch; ++c) p.out[f * ch + c] = pcm_sample(row + static_cast<long long>(c) * p.isz, p.kind, p.isz, p.be);
    }
  }
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
    const int isz = pcm_sample_bytes(it.kind);
    SOME_REQUIRE(isz > 0, "some_pcm_decode_pack: item %d: unknown sample kind %d", i, it.kind);
    SOME_REQUIRE(it.frames >= 0 && it.channels >= 1, "some_pcm_decode_pack: item %d: %lld frames of %d channels", i, it.frames,
                 it.channels);
    SOME_REQUIRE(!it.mono || it.channels <= kMonoMaxChannels,
                 "some_pcm_decode_pack: item %d: a mono down-mix of %d channels (numpy's order is restated up to %d)", i,
                 it.channels, kMonoMaxChannels);
    SOME_REQUIRE(it.frames == 0 || (it.data && it.out), "some_pcm_decode_pack: item %d: null pointer", i);
    const bool be = it.kind == SOME_PCM_S16BE || it.kind == SOME_PCM_S24BE || it.kind == SOME_PCM_S32BE ||
                    it.kind == SOME_PCM_F32BE || it.kind == SOME_PCM_F64BE;
    ps[i] = PcmParams{it.data, it.out, it.frames, it.channels, it.kind, it.mono ? 1 : 0, isz, be ? 1 : 0};
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
