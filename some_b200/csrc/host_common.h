// Host-side helpers shared by the C-ABI entry points: thread-local error string, launch checks and
// TMA tensor-map encoding (cuTensorMapEncodeTiled obtained through cudaGetDriverEntryPoint so the
// library needs no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/some_b200.h"

namespace some {

void set_error(const char* fmt, ...);
int check_launch(const char* what);

// rows x cols bf16 row-major matrix (cols contiguous, `ld` elements between rows); the box is
// box_rows x 64 elements (128 B inner extent) with the 128-byte swizzle the UMMA descriptors expect.
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                      uint32_t box_rows, uint32_t box_cols = 64);

// same for any element size (2 = bf16, 4 = f32): the inner box extent is always 128 bytes (64 bf16 / 32 f32 columns)
int make_tmap_2d(CUtensorMap* out, uint32_t elem_bytes, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_rows, uint32_t box_cols);

// Function attributes (dynamic shared-memory opt-in, carveout) and the SM count are per DEVICE: everything that caches them
// indexes by the current device so that engines on several GPUs of one process work (one slot per device ordinal).
constexpr int kMaxDevices = 64;
int device_index();
int num_sms();

// Programmatic dependent launch (some_set_pdl): a kernel launched through launch_pdl() may become resident while its
// predecessor in the stream is still running; it executes its prologue (barrier init, tensor-map prefetch) and
// blocks in griddep_wait() -- which every such kernel calls before its first access to activations -- until the predecessor has
// completed and flushed.  Pays on small batches, where a step is ~70 dependent launches of a few microseconds each.
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// Workspace carving: consecutive 256-byte aligned buffers of one device block; with base == nullptr it only sizes them.
struct Carver {
  uint8_t* base;
  uint64_t off = 0;
  template <class T>
  T* take(uint64_t bytes) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += (bytes + 255) & ~uint64_t(255);
    return p;
  }
};

#define SOME_REQUIRE(cond, ...)      \
  do {                               \
    if (!(cond)) {                   \
      some::set_error(__VA_ARGS__);  \
      return -1;                     \
    }                                \
  } while (0)

// some_flac_decode, and with `failed` != NULL (a device int, INT_MAX on entry) also the lowest chain index k whose frame failed
// to decode, so that a caller decoding many recordings can name the one that failed.
int flac_decode_chain(const uint8_t* data, const some_flac_stream* streams, const some_flac_frame* frames, const int32_t* chain,
                      const int64_t* scratch_off, const int64_t* out_off, int n_chain, int32_t* scratch, float* out, int mono,
                      int* status, int* failed, cudaStream_t stream);

// The bytes of one sample of a SOME_PCM_* kind (0: not a kind).
inline int pcm_sample_bytes(int kind) {
  switch (kind) {
    case SOME_PCM_U8: case SOME_PCM_S8: case SOME_PCM_ULAW: case SOME_PCM_ALAW: return 1;
    case SOME_PCM_S16: case SOME_PCM_S16BE: return 2;
    case SOME_PCM_S24: case SOME_PCM_S24BE: return 3;
    case SOME_PCM_S32: case SOME_PCM_S32BE: case SOME_PCM_F32: case SOME_PCM_F32BE: return 4;
    case SOME_PCM_F64: case SOME_PCM_F64BE: return 8;
    default: return 0;
  }
}

// The number of RMS frames whose windows end within the first `fixed` samples (the streaming slicer and the stream).
inline int64_t frames_within(const some_slicer_frames& f, int64_t fixed) {
  const int64_t reach = f.win_size - f.win_size / 2;          // frame k reads samples up to k hop - win / 2 + win - 1
  return fixed < reach ? 0 : (fixed - reach) / f.hop_size + 1;
}

// The RMS frames slicer2 cuts a whole recording of n samples by (librosa's centred frames), or 0 when the recording is one
// chunk anyway: no longer than min_length hops (slicer2.py:79-80).
inline int64_t frames_whole(const some_slicer_frames& f, int64_t n) {
  if ((n + f.hop_size - 1) / f.hop_size <= f.min_length) return 0;
  return 1 + (n + 2 * (f.win_size / 2) - f.win_size) / f.hop_size;
}

// Packed descriptors of a many-window launch (some_resample_windows_pack, some_slicer_rms_windows_pack and the stream's
// upload): a header, the windows' first tiles (K + 1 prefix sums: the grid lays the windows' tiles end to end) and the K
// kernel parameter blocks P, each part 16-byte aligned.  The host copy sizes the launch; the kernel reads a device copy of
// the same bytes.
struct WindowsHeader {
  long long K, tiles, smem, pad;
};
constexpr size_t align16(size_t b) { return (b + 15) & ~size_t(15); }
template <class P>
size_t windows_bytes(int K) {
  return sizeof(WindowsHeader) + align16(8ull * (K + 1)) + sizeof(P) * K;
}
inline long long* windows_tile0(void* desc) {
  return reinterpret_cast<long long*>(static_cast<char*>(desc) + sizeof(WindowsHeader));
}
template <class P>
P* windows_params(void* desc, int K) {
  return reinterpret_cast<P*>(static_cast<char*>(desc) + sizeof(WindowsHeader) + align16(8ull * (K + 1)));
}

// Completes the descriptors of K windows whose tile counts the packer left in tile0[1 .. K]: the prefix sums and the header.
inline void windows_index(void* desc, int K, long long smem) {
  WindowsHeader* h = static_cast<WindowsHeader*>(desc);
  long long* tile0 = windows_tile0(desc);
  tile0[0] = 0;
  for (int w = 0; w < K; ++w) tile0[w + 1] += tile0[w];
  h->K = K, h->tiles = tile0[K], h->smem = smem, h->pad = 0;
}

// The window w with tile0[w] <= tile < tile0[w + 1]: the last of equal prefixes, so windows without tiles are skipped.
__device__ __forceinline__ int window_of(const long long* __restrict__ tile0, int K, long long tile) {
  int lo = 0, hi = K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) / 2;
    if (__ldg(tile0 + mid) <= tile) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

}  // namespace some
