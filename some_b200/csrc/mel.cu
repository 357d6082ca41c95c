// K-mel: fused zero-pad + framing + periodic-Hann window + 2048-point real FFT + magnitude + sparse
// triangular mel filterbank + log(clamp) -> [M, 80], written frame-major so the reference's
// `.transpose(1, 2)` (inference/me_infer.py:31) disappears.  Restates modules/rmvpe/spec.py:38-72
// (keyshift = 0, speed = 1, center = True).
//
// ONE WARP PER FRAME, the FFT in registers (round 1 ran five radix-4 stages through shared memory with a CTA barrier after
// each: 1.45 ms per 64 x 30 s batch, 4 % of the HBM rate).  The 2048 real samples are packed as 1024 complex points
// z[n] = w[2n] x[2n] + i w[2n+1] x[2n+1] and transformed as 32 x 32 (Cooley-Tukey, n = 32 n1 + n2, k = k1 + 32 k2):
//   1. lane n2 loads z[32 n1 + n2], n1 < 32 (coalesced 8-byte loads straight from the waveform; samples outside [0, L) read
//      as zero = the reference's F.pad 1024 / 1024) and runs a 32-point radix-2 DIF DFT over n1 in registers;
//   2. times W_1024^(n2 k1) (table [k1][n2], conflict-free), transposed through a warp-private 8 KB XOR-swizzled tile;
//   3. lane k1 runs the second 32-point DFT over n2 -> Z[k1 + 32 k2], written back to the tile in natural order;
//   4. real-FFT unpack for bins 0..371 only (mel weights above 8 kHz are zero), |X| -> the tile (as floats);
//   5. mel[m] = sum over the filter's contiguous bin range (<= 24 bins), log(max(., clamp)); lane m, m + 32, m + 64.
// No CTA barrier after the table load; a CTA is just MEL_WARPS independent warps sharing the 19 KB of tables.
// Algorithmic traffic: 512 x 4 B in + 80 x 4 B out per frame (2368 B); ~60 kFLOP per frame keep it issue-bound.
// On an H100 80GB HBM3 (700 W) one 64 x 30 s batch takes 0.61 ms (bench_rowwise.py); while c[] of the DFTs sat in local
// memory (a 336-byte stack frame and spills, see dif_butterflies) it took 3.67 ms.
#include "host_common.h"
#include "sm90_ptx.cuh"

#include "../../include/some_b200.h"

namespace some {

constexpr int MEL_WARPS = 8;                   // warps per CTA
constexpr int MEL_FPW = 8;                     // consecutive frames per warp (75 % of a frame's samples are L1 hits)
constexpr int MEL_FPB = MEL_WARPS * MEL_FPW;   // frames per CTA
constexpr int MEL_MAXW = SOME_MEL_MAXW;
constexpr int MEL_TW = SOME_MEL_TW;            // 1024 inter-pass twiddles [k1][n2] + 372 unpack twiddles
constexpr int MEL_WSTRIDE = 96;                // filters padded to 96 per tap row: lanes m, m + 32, m + 64 read consecutive words
constexpr int MEL_SMEM = MEL_TW * 8 + 2048 * 4 /*window*/ + SOME_MEL_MAXW * MEL_WSTRIDE * 4 /*mel weights [tap][filter]*/ +
                         MEL_WARPS * 1024 * 8 /*tiles*/;

struct cpx {
  float x, y;
};
__device__ __forceinline__ cpx cadd(cpx a, cpx b) { return {a.x + b.x, a.y + b.y}; }
__device__ __forceinline__ cpx csub(cpx a, cpx b) { return {a.x - b.x, a.y - b.y}; }
__device__ __forceinline__ cpx cmul(cpx a, float wr, float wi) { return {a.x * wr - a.y * wi, a.x * wi + a.y * wr}; }

// W_32^j = exp(-2 pi i j / 32), j < 16 (rounded from double)
__device__ constexpr float kC32[16] = {1.0f,          0.98078528f,  0.92387953f,  0.83146961f, 0.70710678f,  0.55557023f,
                                       0.38268343f,   0.19509032f,  0.0f,         -0.19509032f, -0.38268343f, -0.55557023f,
                                       -0.70710678f,  -0.83146961f, -0.92387953f, -0.98078528f};
__device__ constexpr float kS32[16] = {0.0f,          -0.19509032f, -0.38268343f, -0.55557023f, -0.70710678f, -0.83146961f,
                                       -0.92387953f,  -0.98078528f, -1.0f,        -0.98078528f, -0.92387953f, -0.83146961f,
                                       -0.70710678f,  -0.55557023f, -0.38268343f, -0.19509032f};

// Twiddle multiply of a DFT butterfly, W_32^t with T = t known at compile time, its rounding spelled out so that it does
// not depend on how the compiler contracts the products (that changes with whether the twiddle is a constant or a load):
// re = fma(x, wr, -(y wi)), im = fma(y, wr, x wi).  For W_32^12 in the span-4 stage, where wr = wi, the product x wr is
// the one that is rounded: re = fma(y, -wi, x wr).  These are the roundings of the earlier form of this kernel, kept so
// that its outputs stay the same bits.
template <int HALF, int T>
__device__ __forceinline__ cpx twiddle(cpx d) {
  const float wr = kC32[T], wi = kS32[T];
  if (HALF == 4 && T == 12) return {__fmaf_rn(d.y, -wi, __fmul_rn(d.x, wr)), __fmaf_rn(d.y, wr, __fmul_rn(d.x, wi))};
  return {__fmaf_rn(d.x, wr, -__fmul_rn(d.y, wi)), __fmaf_rn(d.y, wr, __fmul_rn(d.x, wi))};
}
// One radix-2 DIF stage of butterflies HALF apart.  HALF and j are template arguments, so every register index and twiddle
// is a compile-time constant: with the stage span derived from an unrolled outer loop instead, the compiler unrolled the
// inner loop by 4 before the outer one, indexed c[] at run time and put it in local memory.
template <int HALF, int J = 0>
__device__ __forceinline__ void dif_butterflies(cpx (&c)[32], int g) {
  if constexpr (J < HALF) {
    const cpx a = c[g + J], b = c[g + J + HALF];
    c[g + J] = cadd(a, b);
    const cpx d = csub(a, b);
    constexpr int t = J * (16 / HALF);   // W_(2 HALF)^J = W_32^t
    if constexpr (t == 0) {
      c[g + J + HALF] = d;
    } else if constexpr (t == 8) {       // -i
      c[g + J + HALF] = {d.y, -d.x};
    } else {
      c[g + J + HALF] = twiddle<HALF, t>(d);
    }
    dif_butterflies<HALF, J + 1>(c, g);
  }
}
template <int HALF>
__device__ __forceinline__ void dif_stage(cpx (&c)[32]) {
#pragma unroll
  for (int g = 0; g < 32; g += 2 * HALF) dif_butterflies<HALF>(c, g);
}
// In-place 32-point radix-2 DIF DFT, fully unrolled: c[i] ends up holding X[bitrev5(i)].
__device__ __forceinline__ void dft32(cpx (&c)[32]) {
  dif_stage<16>(c);
  dif_stage<8>(c);
  dif_stage<4>(c);
  dif_stage<2>(c);
  dif_stage<1>(c);
}
__device__ __forceinline__ constexpr int bitrev5(int i) {
  return ((i & 1) << 4) | ((i & 2) << 2) | (i & 4) | ((i & 8) >> 2) | ((i & 16) >> 4);
}
// warp-private 32 x 32 complex tile, element (row, col) with the column XOR-swizzled by the row: a lane writing its 32
// values down a column and a lane reading its 32 values along a row are both conflict-free (8-byte accesses, half-warps)
__device__ __forceinline__ int tsw(int row, int col) { return row * 32 + (col ^ row); }
// The lane index, read afresh where it is called: the 64 swizzled tile addresses of steps 2 and 3 are then formed in each
// frame next to their use instead of being hoisted out of the frame loop, where they held ~40 registers for the whole
// kernel and pushed it into spills at the register budget of 3 CTAs per SM.
__device__ __forceinline__ int lane_now() {
  int l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}

// 2 CTAs x 8 warps per SM: at most 128 registers per thread (no stack frame, no spills) and 2 x 92 KB of shared
// memory, which needs the maximum shared-memory carveout (set at the first launch, checked with the occupancy calculator).
#ifndef MEL_MIN_CTAS
#define MEL_MIN_CTAS 2
#endif
__global__ void __launch_bounds__(MEL_WARPS * 32, MEL_MIN_CTAS)
mel_kernel(const float* __restrict__ wave, const int64_t* __restrict__ clip_start, const int64_t* __restrict__ clip_len,
           const int32_t* __restrict__ cu_frames,
           int tiles_per_clip, const int32_t* __restrict__ mel_start, const int32_t* __restrict__ mel_count,
           const float* __restrict__ mel_weights, const float* __restrict__ twiddle, const float* __restrict__ window,
           float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16, float clamp) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);             // [1024] W_1024^(n2 k1) at [k1 * 32 + n2], then [372] W_2048^k
  float* s_win = reinterpret_cast<float*>(s_tw + MEL_TW);
  float* s_mw = s_win + 2048;                                      // [MEL_MAXW][MEL_WSTRIDE], zero beyond a filter's width
  float2* s_tiles = reinterpret_cast<float2*>(s_mw + MEL_MAXW * MEL_WSTRIDE);

  const int clip = blockIdx.x / tiles_per_clip;
  const int tile = blockIdx.x - clip * tiles_per_clip;
  const int row_begin = cu_frames[clip];
  const int T = cu_frames[clip + 1] - row_begin;
  const int frame0 = tile * MEL_FPB;
  if (frame0 >= T) return;
  const int64_t L = clip_len[clip];
  const float* __restrict__ x = wave + clip_start[clip];
  const bool vec_ok = ((reinterpret_cast<uintptr_t>(x) & 7) == 0);

  for (int i = threadIdx.x; i < MEL_TW; i += MEL_WARPS * 32) s_tw[i] = reinterpret_cast<const float2*>(twiddle)[i];
  for (int i = threadIdx.x; i < 2048; i += MEL_WARPS * 32) s_win[i] = window[i];
  for (int i = threadIdx.x; i < MEL_MAXW * MEL_WSTRIDE; i += MEL_WARPS * 32) {
    const int j = i / MEL_WSTRIDE, m = i - j * MEL_WSTRIDE;
    s_mw[i] = (m < SOME_N_MELS && j < __ldg(mel_count + m)) ? __ldg(mel_weights + m * MEL_MAXW + j) : 0.f;
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float2* tile_z = s_tiles + warp * 1024;
  float* mag = reinterpret_cast<float*>(tile_z);
  // mel filters of this lane: m = lane, lane + 32, lane + 64 (< 80); first bin of each
  int m_st[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int m = lane + 32 * i;
    m_st[i] = m < SOME_N_MELS ? __ldg(mel_start + m) : 0;
  }

  for (int fi = 0; fi < MEL_FPW; ++fi) {
    const int f = frame0 + warp * MEL_FPW + fi;
    if (f >= T) break;   // warp-uniform
    // ---- 1. load + window + first DFT (over n1, lane = n2).  All 32 loads of a lane are independent and issued back to
    //         back (one memory round trip per frame); frames that touch the zero padding take the predicated form.
    cpx c[32];
    const int64_t s0 = static_cast<int64_t>(f) * 512 - 1024 + 2 * lane;   // sample index of z[n2]'s real part for n1 = 0
    const bool interior = vec_ok && f >= 2 && (static_cast<int64_t>(f) * 512 + 1024 <= L);   // warp-uniform
    if (interior) {
#pragma unroll
      for (int n1 = 0; n1 < 32; ++n1) {
        const float2 xv = __ldg(reinterpret_cast<const float2*>(x + s0 + 64 * n1));
        c[n1] = {xv.x, xv.y};
      }
    } else {
      // edge frame (or unaligned clip): stage the 2048 samples through the warp's tile with the zero padding applied
      __syncwarp();   // the previous frame's mel pass has finished reading the tile
      float* stage = reinterpret_cast<float*>(tile_z);
      const int64_t base = static_cast<int64_t>(f) * 512 - 1024;
      for (int i = lane; i < 2048; i += 32) {
        const int64_t sidx = base + i;
        stage[i] = (sidx >= 0 && sidx < L) ? __ldg(x + sidx) : 0.f;
      }
      __syncwarp();
#pragma unroll
      for (int n1 = 0; n1 < 32; ++n1) {
        const float2 xv = *reinterpret_cast<const float2*>(stage + 64 * n1 + 2 * lane);
        c[n1] = {xv.x, xv.y};
      }
    }
#pragma unroll
    for (int n1 = 0; n1 < 32; ++n1) {
      const float2 wv = *reinterpret_cast<const float2*>(s_win + 64 * n1 + 2 * lane);
      c[n1].x = __fmul_rn(c[n1].x, wv.x);   // a rounded product: not fused into the first butterfly's add
      c[n1].y = __fmul_rn(c[n1].y, wv.y);
    }
    dft32(c);
    // ---- 2. twiddle W_1024^(n2 k1) and transpose: register i holds k1 = bitrev5(i)
    __syncwarp();   // the previous frame's mel pass has finished reading the tile
    const int ln = lane_now();
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int k1 = bitrev5(i);
      const float2 w = s_tw[k1 * 32 + ln];
      const cpx v = cmul(c[i], w.x, w.y);
      tile_z[tsw(k1, ln)] = make_float2(v.x, v.y);
    }
    __syncwarp();
    // ---- 3. second DFT (over n2, lane = k1)
#pragma unroll
    for (int n2 = 0; n2 < 32; ++n2) {
      const float2 v = tile_z[tsw(ln, n2)];
      c[n2] = {v.x, v.y};
    }
    dft32(c);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 32; ++i) tile_z[lane + 32 * bitrev5(i)] = make_float2(c[i].x, c[i].y);   // Z[k1 + 32 k2], natural order
    __syncwarp();
    // ---- 4. real-FFT unpack, bins 0..371:  X[k] = E + W_2048^k O,  E = (Z[k] + conj Z[N-k]) / 2,
    //         O = -i (Z[k] - conj Z[N-k]) / 2;  all reads first, then the magnitudes overwrite the tile
    float mg[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) {
      const int k = lane + 32 * i;
      mg[i] = 0.f;
      if (k < SOME_MEL_BINS) {
        const float2 zk = tile_z[k];
        const float2 zn = tile_z[(1024 - k) & 1023];
        const float ex = 0.5f * (zk.x + zn.x), ey = 0.5f * (zk.y - zn.y);
        const float dx = zk.x - zn.x, dy = zk.y + zn.y;   // Z[k] - conj(Z[N-k])
        const float ox = 0.5f * dy, oy = -0.5f * dx;      // -i/2 * that
        const float2 w = s_tw[1024 + k];                  // W_2048^k
        const float re = ex + (w.x * ox - w.y * oy), im = ey + (w.x * oy + w.y * ox);
        mg[i] = sqrtf(re * re + im * im);
      }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 12; ++i) {
      const int k = lane + 32 * i;
      if (k < SOME_MEL_BINS) mag[k] = mg[i];
    }
    __syncwarp();
    // ---- 5. mel + log
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int m = lane + 32 * i;
      if (m < SOME_N_MELS) {
        // all MEL_MAXW taps, unrolled: the weights beyond the filter's width are zero (the bin index is clamped so that the
        // zero always multiplies a finite magnitude); ascending bins, one fma chain = the order of the round-1 kernel
        // (st is made opaque per frame so that the 24 clamped bin addresses are formed here, not kept for the whole loop)
        int st = m_st[i];
        asm volatile("" : "+r"(st));
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < MEL_MAXW; ++j)
          acc = fmaf(s_mw[j * MEL_WSTRIDE + m], mag[min(st + j, SOME_MEL_BINS - 1)], acc);
        const float v = logf(fmaxf(acc, clamp));
        const size_t o = static_cast<size_t>(row_begin + f) * SOME_N_MELS + m;
        if (out_f32 != nullptr) out_f32[o] = v;
        if (out_bf16 != nullptr) out_bf16[o] = __float2bfloat16_rn(v);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// K-mel-keyshift (SURVEY.md §8f-4): the key-shift / speed path of MelSpectrogram.forward (modules/rmvpe/spec.py:39-46,
// 63-68), used by the binarizer's pitch augmentation (preprocessing/me_binarizer.py:235-247).  The STFT length becomes
// n_fft' = round(2048 * 2^(keyshift / 12)) — an arbitrary integer, so no radix FFT — but only bins 0..371 of it reach the
// mel filterbank: they are evaluated as a direct DFT in fp32 with an exact twiddle table exp(-2 pi i m / n_fft') indexed by
// (k n) mod n_fft' (no recurrences, no phase drift), |X| scaled by win_length / win_length' (spec.py:68), then the same
// sparse filterbank + log.  CTA = KS_FR consecutive frames of one clip x 384 threads (thread = bin); the samples the
// frames cover are staged once in shared memory, the window is applied on the fly.
constexpr int KS_FR = 8;            // frames per CTA
constexpr int KS_THREADS = 384;     // >= SOME_MEL_BINS

__global__ void __launch_bounds__(KS_THREADS)
mel_dft_kernel(const float* __restrict__ wave, const int64_t* __restrict__ clip_start, const int64_t* __restrict__ clip_len,
               const int32_t* __restrict__ cu_frames, int tiles_per_clip, int n_fft, int hop, int pad_left, float mag_scale,
               const int32_t* __restrict__ mel_start, const int32_t* __restrict__ mel_count,
               const float* __restrict__ mel_weights, const float* __restrict__ twiddle, const float* __restrict__ window,
               float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_bf16, float clamp) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float2* s_tw = reinterpret_cast<float2*>(smem_raw);                 // [n_fft]
  float* s_win = reinterpret_cast<float*>(s_tw + n_fft);              // [n_fft]
  float* s_x = s_win + n_fft;                                         // [n_fft + (KS_FR - 1) * hop]
  float* s_mag = s_x + n_fft + (KS_FR - 1) * hop;                     // [KS_FR][SOME_MEL_BINS]

  const int clip = blockIdx.x / tiles_per_clip;
  const int tile = blockIdx.x - clip * tiles_per_clip;
  const int row_begin = cu_frames[clip];
  const int T = cu_frames[clip + 1] - row_begin;
  const int frame0 = tile * KS_FR;
  if (frame0 >= T) return;
  const int64_t L = clip_len[clip];
  const float* __restrict__ x = wave + clip_start[clip];
  const int nframes = min(KS_FR, T - frame0);
  const int span = n_fft + (KS_FR - 1) * hop;
  const int64_t s0 = static_cast<int64_t>(frame0) * hop - pad_left;   // F.pad(pad_left, pad_right) of spec.py:47-50
  for (int i = threadIdx.x; i < span; i += KS_THREADS) {
    const int64_t si = s0 + i;
    s_x[i] = (si >= 0 && si < L) ? x[si] : 0.f;
  }
  for (int i = threadIdx.x; i < n_fft; i += KS_THREADS) {
    s_tw[i] = reinterpret_cast<const float2*>(twiddle)[i];
    s_win[i] = window[i];
  }
  __syncthreads();

  const int k = threadIdx.x;
  if (k < SOME_MEL_BINS) {
    float re[KS_FR], im[KS_FR];
#pragma unroll
    for (int f = 0; f < KS_FR; ++f) re[f] = im[f] = 0.f;
    int idx = 0;   // (k * n) mod n_fft
    for (int n = 0; n < n_fft; ++n) {
      const float2 w = s_tw[idx];
      const float wn = s_win[n];
#pragma unroll
      for (int f = 0; f < KS_FR; ++f) {
        const float v = s_x[f * hop + n] * wn;
        re[f] = fmaf(v, w.x, re[f]);
        im[f] = fmaf(v, w.y, im[f]);
      }
      idx += k;
      if (idx >= n_fft) idx -= n_fft;
    }
    const bool have_bin = k < n_fft / 2 + 1;   // spec.py:65-67: bins the shorter FFT does not have are zero
#pragma unroll
    for (int f = 0; f < KS_FR; ++f)
      s_mag[f * SOME_MEL_BINS + k] = have_bin ? sqrtf(re[f] * re[f] + im[f] * im[f]) * mag_scale : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nframes * SOME_N_MELS; i += KS_THREADS) {
    const int f = i / SOME_N_MELS, m = i - f * SOME_N_MELS;
    const int st = __ldg(mel_start + m), cn = __ldg(mel_count + m);
    float acc = 0.f;
    for (int j = 0; j < cn; ++j) acc = fmaf(__ldg(mel_weights + m * MEL_MAXW + j), s_mag[f * SOME_MEL_BINS + st + j], acc);
    const float v = logf(fmaxf(acc, clamp));
    const size_t o = static_cast<size_t>(row_begin + frame0 + f) * SOME_N_MELS + m;
    if (out_f32 != nullptr) out_f32[o] = v;
    if (out_bf16 != nullptr) out_bf16[o] = __float2bfloat16_rn(v);
  }
}

}  // namespace some

using namespace some;

extern "C" int some_mel_logmel(const float* wave, const int64_t* clip_start, const int64_t* clip_len,
                               const int32_t* cu_frames, int B,
                               int max_frames, const int32_t* mel_start, const int32_t* mel_count,
                               const float* mel_weights, const float* twiddle, const float* window, float* out_f32,
                               uint16_t* out_bf16, float clamp, cudaStream_t stream) {
  SOME_REQUIRE(wave && clip_start && clip_len && cu_frames && mel_start && mel_count && mel_weights && twiddle && window,
               "some_mel_logmel: null pointer");
  SOME_REQUIRE(out_f32 || out_bf16, "some_mel_logmel: no output buffer");
  if (B <= 0 || max_frames <= 0) return 0;
  static bool configured[kMaxDevices] = {};   // function attributes are per device
  const int dev_ = device_index();
  if (!configured[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MEL_SMEM);
    SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(mel): %s", cudaGetErrorString(e));
    e = cudaFuncSetAttribute(mel_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(mel carveout): %s", cudaGetErrorString(e));
    int ctas = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, mel_kernel, MEL_WARPS * 32, MEL_SMEM);
    SOME_REQUIRE(e == cudaSuccess && ctas >= MEL_MIN_CTAS, "some_mel_logmel: %d CTAs per SM, the kernel is built for %d (%s)",
                 ctas, MEL_MIN_CTAS, cudaGetErrorString(e));
    configured[dev_] = true;
  }
  const int tiles_per_clip = (max_frames + MEL_FPB - 1) / MEL_FPB;
  const long long grid = 1ll * tiles_per_clip * B;
  SOME_REQUIRE(grid < (1ll << 31), "some_mel_logmel: grid too large");
  mel_kernel<<<static_cast<unsigned>(grid), MEL_WARPS * 32, MEL_SMEM, stream>>>(
      wave, clip_start, clip_len, cu_frames, tiles_per_clip, mel_start, mel_count, mel_weights, twiddle, window, out_f32,
      reinterpret_cast<__nv_bfloat16*>(out_bf16), clamp);
  return check_launch("some_mel_logmel");
}

extern "C" int some_mel_logmel_keyshift(const float* wave, const int64_t* clip_start, const int64_t* clip_len,
                                        const int32_t* cu_frames, int B, int max_frames, int n_fft, int hop, int pad_left,
                                        float mag_scale, const int32_t* mel_start, const int32_t* mel_count,
                                        const float* mel_weights, const float* twiddle, const float* window, float* out_f32,
                                        uint16_t* out_bf16, float clamp, cudaStream_t stream) {
  SOME_REQUIRE(wave && clip_start && clip_len && cu_frames && mel_start && mel_count && mel_weights && twiddle && window,
               "some_mel_logmel_keyshift: null pointer");
  SOME_REQUIRE(out_f32 || out_bf16, "some_mel_logmel_keyshift: no output buffer");
  SOME_REQUIRE(n_fft >= SOME_MEL_BINS && n_fft <= 8192 && hop >= 1 && hop <= 4096 && pad_left >= 0,
               "some_mel_logmel_keyshift: n_fft %d / hop %d / pad %d out of range", n_fft, hop, pad_left);
  if (B <= 0 || max_frames <= 0) return 0;
  const int smem = n_fft * 8 + n_fft * 4 + (n_fft + (KS_FR - 1) * hop) * 4 + KS_FR * SOME_MEL_BINS * 4;
  SOME_REQUIRE(smem <= 227 * 1024, "some_mel_logmel_keyshift: n_fft %d with hop %d needs %d B of shared memory", n_fft, hop, smem);
  cudaError_t e = cudaFuncSetAttribute(mel_dft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(mel_dft): %s", cudaGetErrorString(e));
  const int tiles_per_clip = (max_frames + KS_FR - 1) / KS_FR;
  const long long grid = 1ll * tiles_per_clip * B;
  SOME_REQUIRE(grid < (1ll << 31), "some_mel_logmel_keyshift: grid too large");
  mel_dft_kernel<<<static_cast<unsigned>(grid), KS_THREADS, smem, stream>>>(
      wave, clip_start, clip_len, cu_frames, tiles_per_clip, n_fft, hop, pad_left, mag_scale, mel_start, mel_count, mel_weights,
      twiddle, window, out_f32, reinterpret_cast<__nv_bfloat16*>(out_bf16), clamp);
  return check_launch("some_mel_logmel_keyshift");
}
