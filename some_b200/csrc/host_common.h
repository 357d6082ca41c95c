// Host-side helpers shared by the C-ABI entry points: thread-local error string, launch checks and
// TMA tensor-map encoding (cuTensorMapEncodeTiled obtained through cudaGetDriverEntryPoint so the
// library needs no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

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

#define SOME_REQUIRE(cond, ...)      \
  do {                               \
    if (!(cond)) {                   \
      some::set_error(__VA_ARGS__);  \
      return -1;                     \
    }                                \
  } while (0)

}  // namespace some
