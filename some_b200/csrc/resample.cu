// K-resample: librosa.resample(y, orig_sr, target_sr, res_type='kaiser_best') = resampy.resample(..., filter='kaiser_best') +
// fix_length, as librosa.load calls it for every recording whose rate is not the model's (infer.py:34, batch_infer.py:51,
// webui.py:47; librosa<0.10, requirements.txt:10).  The arithmetic is restated in oracle/resample.py.
//
// Every output sample t is one dot product over at most 2 * (nwin / index_step) taps of a linearly interpolated, tabulated
// Kaiser-windowed sinc.  resampy accumulates it into a float32 output with float64 products: each step is
// y = float32(double(y) + (win[o] + eta * (win[o + 1] - win[o])) * double(x)), left wing first (taps i = 0, 1, ...), then
// the right wing.  Here every one of those operations is an explicitly rounded intrinsic (no FMA contraction), in the same
// order, and all index arithmetic is integer, so the result is BIT-identical to resampy's numba loop.
//
// One CTA computes a tile of RS_TILE consecutive outputs of one recording (thread j owns outputs j, j + 256, ...).  The
// tile's input window (plus the filter half-width on both sides) is staged once in shared memory as float64.  The float64
// table (nwin = 32769 entries, 256 KB) stays in L2; the taps are walked in chunks of RS_CHUNK per wing, and each chunk's
// slice of the table (RS_CHUNK * index_step + 2 entries) is staged in shared memory for the whole tile, so that every tap
// reads shared memory only.  The tile's threads all walk the same chunk sequence; a tap beyond an output's own limit (the
// signal's edges, the end of the table) is skipped, exactly like resampy's loop bounds.
#include <math.h>

#include <algorithm>

#include "host_common.h"

#include "../../include/some_b200.h"

namespace some {

constexpr int RS_THREADS = 256;
constexpr int RS_OPT = 8;                       // outputs per thread
constexpr int RS_TILE = RS_THREADS * RS_OPT;    // outputs per CTA
constexpr int RS_CHUNK = 8;                     // taps per wing per staged table slice
constexpr int RS_NUM_TABLE = 512;               // table entries per zero crossing (resampy's precision = 9)
constexpr int RS_MAX_SMEM = 227 * 1024;

struct ResampleParams {
  const float* x;
  const int64_t* x_start;
  const int64_t* x_len;
  float* y;
  const int64_t* y_start;
  const double* win;
  int nwin;
  int sr_orig, sr_new;
  double ratio;      // float(sr_new) / sr_orig
  double inc;        // 1.0 / ratio: t_out[t] = t * inc
  double scale;      // min(1, ratio)
  int step;          // index_step = int(scale * 512)
  int max_taps;      // nwin / step: the longest wing
  // window variant (one recording, absolute positions): x[i - x_first] is input sample i, y[t - y_first] output t; the
  // outputs [t_begin, t_end) of a recording whose input is `len` samples long (as far as the wing limits see it) are written
  long long x_first, y_first, t_begin, t_end, len;
};

// One wing (left = taps x[n - i], right = x[n + 1 + k]) for this thread's RS_OPT outputs.  xi[k] is the window index of
// x[n] (left) or x[n + 1] (right), lim[k] the number of taps, off / eta the table position of tap 0.
template <bool kLeft>
__device__ __forceinline__ void wing(const ResampleParams& p, double* tab, const double* xs, const int (&xi)[RS_OPT],
                                     const int (&lim)[RS_OPT], const int (&off)[RS_OPT], const double (&eta)[RS_OPT],
                                     float (&acc)[RS_OPT]) {
  const int span = RS_CHUNK * p.step + 2;
  const int n_chunks = (p.max_taps + RS_CHUNK - 1) / RS_CHUNK;
  for (int c = 0; c < n_chunks; ++c) {
    __syncthreads();                                        // the previous slice is no longer read
    const int base = c * RS_CHUNK * p.step;
    for (int j = threadIdx.x; j < span; j += RS_THREADS) {
      const int g = base + j;
      // np.diff(win, append=win[-1]): the last entry's delta is 0, i.e. "win[nwin]" = win[nwin - 1]
      tab[j] = g < p.nwin ? __ldg(p.win + g) : __ldg(p.win + p.nwin - 1);
    }
    __syncthreads();
    // Branch-free: a skipped tap reads entry 0 of both arrays and its result is discarded by a select, so the RS_OPT
    // independent accumulation chains of a thread stay interleaved in the instruction stream.
#pragma unroll
    for (int jj = 0; jj < RS_CHUNK; ++jj) {
      const int i = c * RS_CHUNK + jj;
#pragma unroll
      for (int k = 0; k < RS_OPT; ++k) {
        const bool live = i < lim[k];
        const int o = live ? off[k] + jj * p.step : 0;
        const int xj = live ? (kLeft ? xi[k] - i : xi[k] + i) : 0;
        const double w0 = tab[o], w1 = tab[o + 1];
        const double w = __dadd_rn(w0, __dmul_rn(eta[k], __dsub_rn(w1, w0)));
        const float sum = __double2float_rn(__dadd_rn(static_cast<double>(acc[k]), __dmul_rn(w, xs[xj])));
        acc[k] = live ? sum : acc[k];
      }
    }
  }
}

// table position of a wing's first tap: offset = int(frac * 512), eta = frac * 512 - offset
__device__ __forceinline__ void table_pos(double frac, int& off, double& eta) {
  const double index_frac = __dmul_rn(frac, static_cast<double>(RS_NUM_TABLE));
  off = static_cast<int>(index_frac);
  eta = __dsub_rn(index_frac, static_cast<double>(off));
}

// kWindow = false: the batched form, recording b whole.  kWindow = true: outputs [t_begin, t_end) of one recording from a
// buffer that holds only part of its input.  Every output's arithmetic depends on its absolute position t alone (n, the table
// position, the wing limits against 0 and len), not on the tile it falls in, so both forms, and every kernel that computes
// its tiles with this function, give the same bits.
template <bool kWindow>
__device__ __forceinline__ void resample_tile(const ResampleParams& p, int b, long long tile) {
  extern __shared__ double rs_smem[];
  const long long L = kWindow ? p.len : p.x_len[b];
  const long long n_total = static_cast<long long>(ceil(__dmul_rn(static_cast<double>(L), p.ratio)));   // fix_length
  const long long n_out = L * p.sr_new / p.sr_orig;                                                       // resampy's length
  const long long t0 = (kWindow ? p.t_begin : 0) + tile * RS_TILE;
  const long long t_stop = kWindow ? min(p.t_end, n_total) : n_total;
  if (t0 >= t_stop) return;
  float* y = p.y + (kWindow ? -p.y_first : p.y_start[b]);   // y[t]: output t
  float acc[RS_OPT];
#pragma unroll
  for (int k = 0; k < RS_OPT; ++k) acc[k] = 0.f;

  if (t0 < n_out) {                                         // uniform over the CTA
    const float* x = p.x + (kWindow ? -p.x_first : p.x_start[b]);   // x[i]: input sample i
    double* tab = rs_smem;
    double* xs = rs_smem + RS_CHUNK * p.step + 2;
    const long long t_last = min(t0 + RS_TILE, min(t_stop, n_out)) - 1;
    const long long n_first = static_cast<long long>(__dmul_rn(static_cast<double>(t0), p.inc));
    const long long n_last = static_cast<long long>(__dmul_rn(static_cast<double>(t_last), p.inc));
    const long long lo = max(0ll, n_first - p.max_taps + 1);
    const long long hi = min(L - 1, n_last + p.max_taps);
    for (long long j = threadIdx.x; j <= hi - lo; j += RS_THREADS) xs[j] = static_cast<double>(__ldg(x + lo + j));

    int xi[RS_OPT], lim[RS_OPT], off[RS_OPT];
    double eta[RS_OPT], frac[RS_OPT];
#pragma unroll
    for (int k = 0; k < RS_OPT; ++k) {
      const long long t = t0 + threadIdx.x + k * RS_THREADS;
      const double tr = __dmul_rn(static_cast<double>(t), p.inc);
      const long long n = static_cast<long long>(tr);
      frac[k] = __dmul_rn(p.scale, __dsub_rn(tr, static_cast<double>(n)));
      table_pos(frac[k], off[k], eta[k]);
      xi[k] = static_cast<int>(n - lo);
      lim[k] = t <= t_last ? static_cast<int>(min(n + 1, static_cast<long long>((p.nwin - off[k]) / p.step))) : 0;
    }
    wing<true>(p, tab, xs, xi, lim, off, eta, acc);
#pragma unroll
    for (int k = 0; k < RS_OPT; ++k) {
      const long long t = t0 + threadIdx.x + k * RS_THREADS;
      const long long n = lo + xi[k];
      table_pos(__dsub_rn(p.scale, frac[k]), off[k], eta[k]);
      xi[k] += 1;
      lim[k] = t <= t_last ? static_cast<int>(max(0ll, min(L - n - 1, static_cast<long long>((p.nwin - off[k]) / p.step)))) : 0;
    }
    wing<false>(p, tab, xs, xi, lim, off, eta, acc);
  }
#pragma unroll
  for (int k = 0; k < RS_OPT; ++k) {
    const long long t = t0 + threadIdx.x + k * RS_THREADS;
    if (t < t_stop) y[t] = acc[k];                          // 0 beyond resampy's n_out: fix_length's zero padding
  }
}

template <bool kWindow>
__global__ void __launch_bounds__(RS_THREADS, 2) resample_kaiser_kernel(const ResampleParams p) {
  resample_tile<kWindow>(p, blockIdx.y, blockIdx.x);
}

// K windows of kWindow form in one grid: the windows' tiles laid end to end, each CTA finds its window from the tile prefix.
__global__ void __launch_bounds__(RS_THREADS, 2) resample_windows_kernel(const ResampleParams* __restrict__ ps,
                                                                         const long long* __restrict__ tile0, int K) {
  const long long tile = blockIdx.x;
  const int w = window_of(tile0, K, tile);
  resample_tile<true>(ps[w], 0, tile - tile0[w]);
}


// The rate-pair constants of resampy.resample and the kernel's shared-memory size for them.
int setup(ResampleParams& p, int sr_orig, int sr_new, int nwin, const char* what, double* smem) {
  SOME_REQUIRE(sr_orig > 0 && sr_new > 0, "%s: invalid sample rates %d -> %d", what, sr_orig, sr_new);
  SOME_REQUIRE(nwin >= 2, "%s: table of %d entries", what, nwin);
  p.nwin = nwin;
  p.sr_orig = sr_orig, p.sr_new = sr_new;
  p.ratio = static_cast<double>(sr_new) / static_cast<double>(sr_orig);
  p.inc = 1.0 / p.ratio;
  p.scale = p.ratio < 1.0 ? p.ratio : 1.0;
  p.step = static_cast<int>(p.scale * RS_NUM_TABLE);
  SOME_REQUIRE(p.step >= 1, "%s: %d -> %d is below the table's resolution", what, sr_orig, sr_new);
  p.max_taps = nwin / p.step;
  // input window: n_last - n_first <= ceil((RS_TILE - 1) * inc) + 1, plus the taps on both sides
  const double x_cap = ceil((RS_TILE - 1) * p.inc) + 2.0 * p.max_taps + 4.0;
  *smem = 8.0 * (RS_CHUNK * p.step + 2 + x_cap);
  SOME_REQUIRE(*smem <= RS_MAX_SMEM, "%s: %d -> %d needs %.0f B of shared memory (downsampling by more than "
               "about 11x is not supported)", what, sr_orig, sr_new, *smem);
  return 0;
}

// Output t reads input samples floor(t * inc) - max_taps + 1 .. floor(t * inc) + max_taps (clipped to [0, len)), with
// floor(t * inc) the same double product the kernel forms.
long long centre(const ResampleParams& p, long long t) { return static_cast<long long>(static_cast<double>(t) * p.inc); }

// The outputs [0, *t_end) that `received` input samples fix, and the first input sample outputs from t_begin on read.  While
// the recording may go on (final == 0), an output is fixed when its right wing ends before `received`: then its wing limit
// min(len - n - 1, (nwin - offset) / step) is the table's whatever the final length, and t < received * sr_new / sr_orig
// keeps it below resampy's n_out.  At the end (final != 0) every output up to fix_length's ceil(len * ratio) is fixed.
void plan(const ResampleParams& p, long long received, int final, long long t_begin, long long* t_end, long long* x_first) {
  if (final) {
    *t_end = static_cast<long long>(ceil(static_cast<double>(received) * p.ratio));
  } else {
    const long long last = received - 1 - p.max_taps;       // the largest centre whose right wing is received
    long long t = 0;
    if (last >= 0) {
      t = static_cast<long long>(static_cast<double>(last + 1) * p.ratio);
      while (t > 0 && centre(p, t - 1) > last) --t;         // centre() is monotone in t
      while (centre(p, t) <= last) ++t;
    }
    *t_end = std::min(t, received * p.sr_new / p.sr_orig);
  }
  *x_first = std::max(0ll, centre(p, t_begin) - p.max_taps + 1);
}

// The kernel parameters of one window, with the checks of some_resample_kaiser_window: the buffer must hold every input
// sample the outputs read, and the received input must fix every output requested.
int window_params(const some_resample_window& w, const char* what, ResampleParams& p, double* smem) {
  SOME_REQUIRE(w.x && w.y && w.win, "%s: null pointer", what);
  p = ResampleParams{};
  if (setup(p, w.sr_orig, w.sr_new, w.nwin, what, smem)) return -1;
  long long fixed_end, need_first;
  plan(p, w.received, w.final, w.t_begin, &fixed_end, &need_first);
  SOME_REQUIRE(w.x_first >= 0 && w.x_first <= w.received && w.t_begin >= 0 && w.t_begin <= w.t_end && w.y_first <= w.t_begin,
               "%s: bad window (input from %lld of %lld, outputs [%lld, %lld) at %lld)", what, w.x_first, w.received, w.t_begin,
               w.t_end, w.y_first);
  SOME_REQUIRE(w.t_end <= fixed_end, "%s: outputs up to %lld requested, %lld received input samples fix %lld%s", what, w.t_end,
               w.received, fixed_end, w.final ? "" : " (their right wings would reach past the input)");
  SOME_REQUIRE(w.x_first <= need_first || w.t_begin == w.t_end, "%s: output %lld reads input from %lld, the buffer starts at "
               "%lld", what, w.t_begin, need_first, w.x_first);
  p.x = w.x, p.y = w.y, p.win = w.win;
  p.x_first = w.x_first, p.y_first = w.y_first, p.t_begin = w.t_begin, p.t_end = w.t_end, p.len = w.received;
  return 0;
}

}  // namespace some

using namespace some;

extern "C" int some_resample_kaiser(const float* x, const int64_t* x_start, const int64_t* x_len, float* y,
                                    const int64_t* y_start, int B, long long max_out, int sr_orig, int sr_new,
                                    const double* win, int nwin, cudaStream_t stream) {
  SOME_REQUIRE(x && x_start && x_len && y && y_start && win, "some_resample_kaiser: null pointer");
  SOME_REQUIRE(B >= 0 && B <= 65535 && max_out >= 0, "some_resample_kaiser: bad batch (B %d, max_out %lld)", B, max_out);
  SOME_REQUIRE(sr_orig > 0 && sr_new > 0, "some_resample_kaiser: invalid sample rates %d -> %d", sr_orig, sr_new);
  SOME_REQUIRE(nwin >= 2, "some_resample_kaiser: table of %d entries", nwin);
  if (B == 0 || max_out == 0) return 0;
  ResampleParams p{};
  double smem;
  if (setup(p, sr_orig, sr_new, nwin, "some_resample_kaiser", &smem)) return -1;
  p.x = x, p.x_start = x_start, p.x_len = x_len, p.y = y, p.y_start = y_start, p.win = win;
  const long long tiles = (max_out + RS_TILE - 1) / RS_TILE;
  SOME_REQUIRE(tiles < (1ll << 31), "some_resample_kaiser: grid too large");
  cudaError_t e = cudaFuncSetAttribute(resample_kaiser_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(smem));
  SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(resample): %s", cudaGetErrorString(e));
  resample_kaiser_kernel<false><<<dim3(static_cast<unsigned>(tiles), B), RS_THREADS, static_cast<size_t>(smem), stream>>>(p);
  return check_launch("some_resample_kaiser");
}

extern "C" int some_resample_window_plan(long long received, int final, long long t_begin, int sr_orig, int sr_new, int nwin,
                                         long long* t_end, long long* x_first) {
  SOME_REQUIRE(t_end && x_first && received >= 0 && t_begin >= 0, "some_resample_window_plan: bad arguments");
  ResampleParams p{};
  double smem;
  if (setup(p, sr_orig, sr_new, nwin, "some_resample_window_plan", &smem)) return -1;
  plan(p, received, final, t_begin, t_end, x_first);
  return 0;
}

extern "C" int some_resample_kaiser_window(const float* x, long long x_first, long long received, int final, float* y,
                                           long long y_first, long long t_begin, long long t_end, int sr_orig, int sr_new,
                                           const double* win, int nwin, cudaStream_t stream) {
  const some_resample_window w{x, x_first, received, final, y, y_first, t_begin, t_end, sr_orig, sr_new, win, nwin};
  ResampleParams p;
  double smem;
  if (window_params(w, "some_resample_kaiser_window", p, &smem)) return -1;
  if (t_begin == t_end) return 0;
  const long long tiles = (t_end - t_begin + RS_TILE - 1) / RS_TILE;
  SOME_REQUIRE(tiles < (1ll << 31), "some_resample_kaiser_window: grid too large");
  cudaError_t e = cudaFuncSetAttribute(resample_kaiser_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(smem));
  SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(resample): %s", cudaGetErrorString(e));
  resample_kaiser_kernel<true><<<dim3(static_cast<unsigned>(tiles), 1), RS_THREADS, static_cast<size_t>(smem), stream>>>(p);
  return check_launch("some_resample_kaiser_window");
}

extern "C" long long some_resample_windows_bytes(int K) { return K < 0 ? -1 : static_cast<long long>(windows_bytes<ResampleParams>(K)); }

extern "C" int some_resample_windows_pack(const some_resample_window* w, int K, void* desc) {
  SOME_REQUIRE(desc && K >= 0 && (K == 0 || w), "some_resample_windows_pack: bad arguments");
  char what[64];
  ResampleParams* ps = windows_params<ResampleParams>(desc, K);
  long long* tile0 = windows_tile0(desc);
  double smem_max = 0.0;
  for (int i = 0; i < K; ++i) {
    snprintf(what, sizeof(what), "some_resample_windows_pack: window %d", i);
    double smem;
    if (window_params(w[i], what, ps[i], &smem)) return -1;
    tile0[i + 1] = (w[i].t_end - w[i].t_begin + RS_TILE - 1) / RS_TILE;
    if (tile0[i + 1]) smem_max = std::max(smem_max, smem);
  }
  windows_index(desc, K, static_cast<long long>(smem_max));
  SOME_REQUIRE(windows_tile0(desc)[K] < (1ll << 31), "some_resample_windows_pack: grid too large");
  return 0;
}

extern "C" int some_resample_kaiser_windows(const void* desc, const void* desc_d, cudaStream_t stream) {
  SOME_REQUIRE(desc && desc_d && reinterpret_cast<uintptr_t>(desc_d) % 16 == 0, "some_resample_kaiser_windows: bad arguments");
  const WindowsHeader& h = *static_cast<const WindowsHeader*>(desc);
  if (h.tiles == 0) return 0;
  const int K = static_cast<int>(h.K);
  void* d = const_cast<void*>(desc_d);
  cudaError_t e = cudaFuncSetAttribute(resample_windows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(h.smem));
  SOME_REQUIRE(e == cudaSuccess, "cudaFuncSetAttribute(resample): %s", cudaGetErrorString(e));
  resample_windows_kernel<<<static_cast<unsigned>(h.tiles), RS_THREADS, static_cast<size_t>(h.smem), stream>>>(
      windows_params<ResampleParams>(d, K), windows_tile0(d), K);
  return check_launch("some_resample_kaiser_windows");
}
