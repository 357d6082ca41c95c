// The silence slicer (utils/slicer2.py): where a recording is cut.  Two halves, both bit-exact with the reference.
//
// Device: K-rms, the short-time RMS of a device-resident waveform (slicer2.py:5-38 `get_rms`, called from Slicer.slice :81
// with frame_length = win_size, hop_length = hop_size, constant (zero) padding of frame_length / 2).  The slicer compares
// every RMS value with a threshold and takes argmins over RMS windows (slicer2.py:84-133), so chunk boundaries are only
// reproducible if the RMS values are BIT-identical to numpy's.  numpy reduces the squared window along its contiguous axis
// with pairwise summation (float32): blocks of <= 128 elements are summed with 8 interleaved accumulators combined as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) plus a sequential tail, larger ranges are split at n/2 rounded down to a multiple of 8.
// This kernel evaluates exactly that tree per frame (one thread per frame, no FMA contraction: __fmul_rn / __fadd_rn /
// __fdiv_rn / __fsqrt_rn), so the host half sees the same numbers as the reference.  13.2 M samples (5 min) -> 15 001
// frames x 3528 samples: ~53 M multiply-adds, L1 / L2 resident.
//
// Host: the slicer's decisions on the RMS list (slicer2.py:62-145), taken per silent run instead of per frame, with no CUDA
// call.  One incremental core (SlicerCore) serves the whole-list call (some_slicer_ranges) and the streaming slicer
// (some_slicer_stream_*), so the cut rules exist once, for the native session, streaming and the Python wrappers
// (some_b200/slicer.py) alike.
#include "host_common.h"

#include <math.h>

#include <algorithm>
#include <utility>
#include <vector>

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

// Frame f of a recording of n_samples samples, wave[s - base] being sample s: its value depends on its absolute index and the
// samples alone, so a window of frames over a buffer holding part of the recording gives the whole-recording bits.  Not
// inlined: inlined into the kernels, ptxas unrolled the block sums less (29 global loads instead of 53).
__device__ __noinline__ float rms_frame(const float* __restrict__ wave, long long base, long long n_samples, int frame_length,
                                        int hop, long long f) {
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
  return __fsqrt_rn(__fdiv_rn(total, static_cast<float>(frame_length)));
}

// Frames [f_begin, f_begin + n_frames) into rms[0, n_frames).
__global__ void __launch_bounds__(128) slicer_rms_kernel(const float* __restrict__ wave, long long base, long long n_samples,
                                                         int frame_length, int hop, float* __restrict__ rms, long long f_begin,
                                                         int n_frames) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_frames) return;
  rms[i] = rms_frame(wave, base, n_samples, frame_length, hop, f_begin + i);
}

// One frame window of the many-window launch: the arguments of slicer_rms_kernel.
struct RmsParams {
  const float* wave;
  long long base, n_samples;
  float* rms;
  long long f_begin;
  int frame_length, hop, n_frames, pad;
};
constexpr int RMS_TILE = 128;   // frames per CTA, one thread each

// K frame windows in one grid: the windows' tiles of RMS_TILE frames laid end to end.
__global__ void __launch_bounds__(RMS_TILE) slicer_rms_windows_kernel(const RmsParams* __restrict__ ps,
                                                                      const long long* __restrict__ tile0, int K) {
  const long long tile = blockIdx.x;
  const int w = window_of(tile0, K, tile);
  const RmsParams& p = ps[w];
  const int i = static_cast<int>(tile - tile0[w]) * RMS_TILE + threadIdx.x;
  if (i >= p.n_frames) return;
  p.rms[i] = rms_frame(p.wave, p.base, p.n_samples, p.frame_length, p.hop, p.f_begin + i);
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

namespace {
// The kernel arguments of one frame window, with the checks of some_slicer_rms_window: the buffer must hold every sample
// inside the recording the frames read.
int rms_window_params(const some_rms_window& w, const char* what, RmsParams& p) {
  SOME_REQUIRE(w.wave && w.rms, "%s: null pointer", what);
  SOME_REQUIRE(w.base >= 0 && w.held >= 0 && w.n_samples >= -1 && w.frame_length >= 1 && w.hop >= 1 && w.f_begin >= 0 &&
                   w.f_end >= w.f_begin && w.f_end - w.f_begin < (1ll << 31),
               "%s: bad sizes", what);
  p = RmsParams{w.wave, w.base, 0, w.rms, w.f_begin, w.frame_length, w.hop, static_cast<int>(w.f_end - w.f_begin), 0};
  if (w.f_end == w.f_begin) return 0;
  const long long half = w.frame_length / 2;
  const bool final = w.n_samples >= 0;
  if (final) {
    const long long padded = w.n_samples + 2 * half;
    SOME_REQUIRE(padded >= w.frame_length && w.f_end <= 1 + (padded - w.frame_length) / w.hop,
                 "%s: frame %lld is past the last frame of %lld samples", what, w.f_end - 1, w.n_samples);
  }
  // the samples the frames read that lie inside the recording: the buffer must hold them
  const long long lo = std::max(0ll, w.f_begin * w.hop - half);
  const long long hi = (w.f_end - 1) * w.hop - half + w.frame_length;
  const long long hi_in = final ? std::min(hi, w.n_samples) : hi;
  SOME_REQUIRE(lo >= w.base && hi_in <= w.base + w.held,
               "%s: frames [%lld, %lld) read samples [%lld, %lld), the buffer holds [%lld, %lld)%s", what, w.f_begin, w.f_end, lo,
               hi_in, w.base, w.base + w.held, final ? "" : " (the recording's length is not known yet)");
  p.n_samples = final ? w.n_samples : w.base + w.held;
  return 0;
}
}  // namespace

extern "C" int some_slicer_rms_window(const float* wave, long long base, long long held, long long n_samples, int frame_length,
                                      int hop, float* rms, long long f_begin, long long f_end, cudaStream_t stream) {
  RmsParams p;
  if (rms_window_params({wave, base, held, n_samples, frame_length, hop, rms, f_begin, f_end}, "some_slicer_rms_window", p))
    return -1;
  if (p.n_frames == 0) return 0;
  slicer_rms_kernel<<<static_cast<unsigned>((p.n_frames + 127) / 128), 128, 0, stream>>>(
      p.wave, p.base, p.n_samples, p.frame_length, p.hop, p.rms, p.f_begin, p.n_frames);
  return check_launch("some_slicer_rms_window");
}

extern "C" long long some_slicer_rms_windows_bytes(int K) { return K < 0 ? -1 : static_cast<long long>(windows_bytes<RmsParams>(K)); }

extern "C" int some_slicer_rms_windows_pack(const some_rms_window* w, int K, void* desc) {
  SOME_REQUIRE(desc && K >= 0 && (K == 0 || w), "some_slicer_rms_windows_pack: bad arguments");
  char what[64];
  RmsParams* ps = windows_params<RmsParams>(desc, K);
  long long* tile0 = windows_tile0(desc);
  for (int i = 0; i < K; ++i) {
    snprintf(what, sizeof(what), "some_slicer_rms_windows_pack: window %d", i);
    if (rms_window_params(w[i], what, ps[i])) return -1;
    tile0[i + 1] = (ps[i].n_frames + RMS_TILE - 1) / RMS_TILE;
  }
  windows_index(desc, K, 0);
  SOME_REQUIRE(windows_tile0(desc)[K] < (1ll << 31), "some_slicer_rms_windows_pack: grid too large");
  return 0;
}

extern "C" int some_slicer_rms_windows(const void* desc, const void* desc_d, cudaStream_t stream) {
  SOME_REQUIRE(desc && desc_d && reinterpret_cast<uintptr_t>(desc_d) % 16 == 0, "some_slicer_rms_windows: bad arguments");
  const WindowsHeader& h = *static_cast<const WindowsHeader*>(desc);
  if (h.tiles == 0) return 0;
  const int K = static_cast<int>(h.K);
  void* d = const_cast<void*>(desc_d);
  slicer_rms_windows_kernel<<<static_cast<unsigned>(h.tiles), RMS_TILE, 0, stream>>>(windows_params<RmsParams>(d, K),
                                                                                     windows_tile0(d), K);
  return check_launch("some_slicer_rms_windows");
}

// ---------------------------------------------------------------------------------------------------- slicer decisions
namespace {

// The first index of the minimum of rms[a, min(b, n)) (numpy's argmin: the first NaN wins).  `rms` is a pointer to the whole
// list or a RmsStore of the frames a streaming slicer still holds.
template <class R>
int64_t first_min(const R& rms, int64_t n, int64_t a, int64_t b) {
  b = std::min(b, n);
  int64_t best = a;
  for (int64_t i = a; i < b; ++i) {
    if (isnan(rms[i])) return i;
    if (rms[i] < rms[best]) best = i;
  }
  return best;
}

using Tag = std::pair<int64_t, int64_t>;

// The reference's frame walk (slicer2.py:84-133) for one run of frames with rms < threshold, [s, i): i < total is the
// voiced frame that ends it, i == total a trailing run.  Returns whether the run is cut, with the frames it removes in `tag`.
// Reads rms[s .. s + keep] and rms[max(s, i - keep) .. i] only.
template <class R>
bool run_tag(const R& rms, int64_t total, const some_slicer_frames& f, int64_t s, int64_t i, int64_t& clip_from, Tag& tag) {
  const int64_t keep = f.max_sil_kept;
  if (i == total) {                                       // trailing silence (slicer2.py:129-133)
    if (total - s < f.min_interval) return false;
    tag = {first_min(rms, total, s, std::min(total, s + keep) + 1), total + 1};
    return true;
  }
  const bool leading = s == 0 && i > keep;
  const bool middle = i - s >= f.min_interval && i - clip_from >= f.min_length;
  if (!(leading || middle)) return false;
  const int64_t span = i - s;
  if (span <= keep) {
    const int64_t cut = first_min(rms, total, s, i + 1);
    tag = s == 0 ? Tag(0, cut) : Tag(cut, cut);
    clip_from = cut;
  } else if (span <= 2 * keep) {
    const int64_t mid = first_min(rms, total, i - keep, s + keep + 1);
    const int64_t left = first_min(rms, total, s, s + keep + 1);
    const int64_t right = first_min(rms, total, i - keep, i + 1);
    tag = s == 0 ? Tag(0, right) : Tag(std::min(left, mid), std::max(right, mid));
    clip_from = tag.second;
  } else {
    const int64_t left = first_min(rms, total, s, s + keep + 1);
    const int64_t right = first_min(rms, total, i - keep, i + 1);
    tag = s == 0 ? Tag(0, right) : Tag(left, right);
    clip_from = right;
  }
  return true;
}

// The RMS values run_tag can still read while the list arrives frame by frame: none outside a silent run; inside the run
// that began at frame ss, frames [ss, ss + keep] (`head`, once the run is long) and the last keep + 1 (`tail`), whichever
// frame ends the run.  O(max_sil_kept) values however long the run.
class RmsStore {
 public:
  float operator[](int64_t k) const { return k >= tail_base_ ? tail_[k - tail_base_] : head_[k - head_base_]; }
  void start(int64_t ss) {
    head_.clear(), tail_.clear();
    head_base_ = tail_base_ = ss;
  }
  void push(float v, int64_t keep) {
    tail_.push_back(v);
    const int64_t end = tail_base_ + static_cast<int64_t>(tail_.size());
    const int64_t dead = end - keep - 1 - tail_base_;            // frames before the last keep + 1
    if (dead <= std::max<int64_t>(keep + 1, 64)) return;         // erase in batches
    if (head_.empty()) head_.assign(tail_.begin(), tail_.begin() + keep + 1);   // tail_base_ == ss here
    tail_.erase(tail_.begin(), tail_.begin() + dead);
    tail_base_ += dead;
  }
  size_t size() const { return head_.size() + tail_.size(); }

 private:
  std::vector<float> head_, tail_;
  int64_t head_base_ = 0, tail_base_ = 0;
};

// The reference's cuts (slicer2.py:84-145) on an RMS list that arrives in pieces.  Each range is returned as soon
// as no later frame can change it:
//  (a) when the voiced frame that ends a cut run is known: the run's tag, and with it the end of the range before it;
//  (b) or, for a run that began at ss > 0 and is still silent at frame j = max(ss + 2 keep, ss + min_interval - 1,
//      clip_from + min_length - 1), at frame j.  Every frame i that can still end the run has i - ss > 2 keep, so the run is
//      the third case of run_tag (span > 2 keep) with both of its conditions met (i - ss >= min_interval, i - clip_from >=
//      min_length), and a recording that ends inside the run has total - ss >= min_interval, so the trailing rule cuts it;
//      both cut the run's start at left = first_min(ss, ss + keep + 1), which frames up to j already fix.  (A run from frame
//      0 ends no range: the leading rule's (0, right) and the all-silent trailing cut differ, so it waits for (a).)
// The next range then begins at the run's right cut, which is no earlier than max(ss, i - keep): open_begin().
// A run from frame 0 that has lasted past frame max(keep, min_interval - 1) (leading_tail()) ends in one of two ways: a voiced
// frame i > keep makes it a leading cut (0, right) with right >= i - keep, so the next range begins no earlier than
// known - keep; or the recording ends inside it, and the trailing rule cuts it at left = first_min(0, keep + 1) <= keep, which
// leaves the one range [0, left) (the all-silent recording).  So during a long leading silence a host keeps the last keep
// frames and, apart, the first keep frames, not everything since frame 0.
class SlicerCore {
 public:
  explicit SlicerCore(const some_slicer_frames& f) : f_(f) {}
  // frames known() .. known() + n; appends the frame ranges [a, b) that became final to `out`
  int feed(const float* rms, int64_t n, std::vector<Tag>& out) {
    const int64_t keep = f_.max_sil_kept;
    for (int64_t j = 0; j < n; ++j) {
      const int64_t k = known_++;
      const float v = rms[j];
      if (v < f_.threshold) {
        if (!in_run_) in_run_ = true, ss_ = k, early_ = false, store_.start(k);
        store_.push(v, keep);
        if (!early_ && ss_ > 0 &&
            k >= std::max({ss_ + 2 * keep, ss_ + f_.min_interval - 1, clip_from_ + f_.min_length - 1})) {   // (b)
          early_first_ = first_min(store_, known_, ss_, ss_ + keep + 1);
          emit(early_first_, out);
          early_ = true;
        }
      } else if (in_run_) {                                                                                  // (a)
        store_.push(v, keep);
        if (end_run(k, out)) return -1;
      }
    }
    return 0;
  }
  // the end of the list: the trailing rule and the last range; a range (0, -1) is the whole recording (no cut at all)
  int finish(std::vector<Tag>& out) {
    if (in_run_ && end_run(known_, out)) return -1;
    if (!any_tag_) {
      out.push_back({0, -1});
    } else if (prev_ < known_) {
      out.push_back({prev_, known_});
    }
    return 0;
  }
  int64_t known() const { return known_; }
  // the first frame a range not yet returned may begin at
  int64_t open_begin() const {
    if (in_run_ && early_) return std::max(ss_, known_ - f_.max_sil_kept);
    if (leading_tail()) return known_ - f_.max_sil_kept;
    return any_tag_ ? prev_ : 0;
  }
  // a range [0, a) with a <= max_sil_kept may still come besides those from open_begin() on
  bool leading_tail() const {
    return in_run_ && ss_ == 0 && known_ > f_.max_sil_kept && known_ >= f_.min_interval;
  }
  size_t held() const { return store_.size(); }

 private:
  void emit(int64_t a, std::vector<Tag>& out) {                // slicer2.py:135-145: the frames before a tag starting at a
    if (any_tag_) {
      out.push_back({prev_, a});
    } else if (a > 0) {
      out.push_back({0, a});
    }
  }
  int end_run(int64_t i, std::vector<Tag>& out) {
    Tag tag;
    const bool cut = run_tag(store_, known_, f_, ss_, i, clip_from_, tag);
    SOME_REQUIRE(!early_ || (cut && tag.first == early_first_),
                 "slicer: the run from frame %lld was cut early at %lld, its end gives %lld", (long long)ss_,
                 (long long)early_first_, cut ? (long long)tag.first : -1ll);
    in_run_ = false;
    store_.start(known_);
    if (!cut) return 0;
    if (!early_) emit(tag.first, out);
    any_tag_ = true;
    prev_ = tag.second;
    return 0;
  }
  some_slicer_frames f_;
  RmsStore store_;
  int64_t known_ = 0, clip_from_ = 0, ss_ = 0, early_first_ = 0, prev_ = 0;
  bool in_run_ = false, early_ = false, any_tag_ = false;
};

}  // namespace

extern "C" int some_slicer_derive(int sample_rate, const some_slicer_params* p, some_slicer_frames* out) {
  SOME_REQUIRE(out != nullptr && sample_rate > 0, "some_slicer_derive: bad arguments");
  some_slicer_params d{-40.0, 5000.0, 300.0, 20.0, 1000.0};    // infer.py: Slicer(sr, max_sil_kept=1000)
  if (p) d = *p;
  SOME_REQUIRE(d.min_length_ms >= d.min_interval_ms && d.min_interval_ms >= d.hop_size_ms,
               "some_slicer_derive: the following condition must be satisfied: min_length >= min_interval >= hop_size");
  SOME_REQUIRE(d.max_sil_kept_ms >= d.hop_size_ms,
               "some_slicer_derive: the following condition must be satisfied: max_sil_kept >= hop_size");
  // Slicer.__init__ (slicer2.py:42-60), with Python's round (half to even: rint in the default rounding mode)
  const double sr = sample_rate;
  const double interval = sr * d.min_interval_ms / 1000.0;
  const double hop = rint(sr * d.hop_size_ms / 1000.0);
  SOME_REQUIRE(hop >= 1.0, "some_slicer_derive: hop_size of %g ms is less than one sample", d.hop_size_ms);
  out->threshold = static_cast<float>(pow(10.0, d.threshold_db / 20.0));   // `rms < threshold` compares in float32
  out->hop_size = static_cast<int>(hop);
  out->win_size = static_cast<int>(std::min(rint(interval), 4.0 * hop));
  out->min_length = static_cast<int>(rint(sr * d.min_length_ms / 1000.0 / hop));
  out->min_interval = static_cast<int>(rint(interval / hop));
  out->max_sil_kept = static_cast<int>(rint(sr * d.max_sil_kept_ms / 1000.0 / hop));
  return 0;
}

extern "C" int some_slicer_ranges(const float* rms, int n_frames, long long n_samples, const some_slicer_frames* f,
                                  int64_t* ranges, int capacity, int* count) {
  SOME_REQUIRE((rms != nullptr || n_frames == 0) && f != nullptr && count != nullptr && n_frames >= 0 && n_samples >= 0,
               "some_slicer_ranges: bad arguments");
  SlicerCore core(*f);
  std::vector<Tag> kept;
  if (core.feed(rms, n_frames, kept) || core.finish(kept)) return -1;
  *count = static_cast<int>(kept.size());
  SOME_REQUIRE(ranges != nullptr && capacity >= *count, "some_slicer_ranges: %d ranges do not fit in a capacity of %d", *count,
               capacity);
  const int64_t hop = f->hop_size;
  for (size_t k = 0; k < kept.size(); ++k) {
    if (kept[k].second < 0) {                   // no tags: the whole recording
      ranges[2 * k] = 0, ranges[2 * k + 1] = n_samples;
      continue;
    }
    ranges[2 * k] = kept[k].first * hop;
    ranges[2 * k + 1] = std::min<int64_t>(n_samples, kept[k].second * hop);
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------- streaming slicer
// SlicerCore in samples, with the short-recording rule (slicer2.py:78-79): a recording of no more than min_length hops is one
// chunk, so ranges are held back until more than min_length * hop_size samples are fixed.
struct some_slicer_stream {
  some_slicer_frames f;
  SlicerCore core;
  std::vector<Tag> queued;                // final ranges (frames) held back by the short-recording rule
  std::vector<int64_t> out;               // the sample ranges the last call returned
  int64_t fixed = 0;
  bool finished = false;
  explicit some_slicer_stream(const some_slicer_frames& fr) : f(fr), core(fr) {}
  bool may_slice() const { return fixed > static_cast<int64_t>(f.min_length) * f.hop_size; }
  // the first model-rate sample a range not yet returned may begin at
  int64_t keep_from() const { return may_slice() ? core.open_begin() * f.hop_size : 0; }
  // the samples [0, head()) a range may still need besides those from keep_from() on
  int64_t head() const { return may_slice() && core.leading_tail() ? static_cast<int64_t>(f.max_sil_kept) * f.hop_size : 0; }
  void release(int64_t n_samples) {
    for (const Tag& t : queued) {
      out.push_back(t.first * f.hop_size);
      out.push_back(t.second < 0 ? n_samples : std::min(n_samples, t.second * f.hop_size));
    }
    queued.clear();
  }
};

namespace {
int slicer_feed(some_slicer_stream* st, const float* rms, int64_t n, int64_t fixed) {
  SOME_REQUIRE(!st->finished, "some_slicer_stream_feed: the stream has finished");
  SOME_REQUIRE(fixed >= st->fixed, "some_slicer_stream_feed: fixed went back from %lld to %lld", (long long)st->fixed,
               (long long)fixed);
  const int64_t known = frames_within(st->f, fixed);
  SOME_REQUIRE(st->core.known() + n <= known, "some_slicer_stream_feed: frames up to %lld fed, %lld fixed samples complete %lld",
               (long long)(st->core.known() + n), (long long)fixed, (long long)known);
  st->out.clear();
  if (st->core.feed(rms, n, st->queued)) return -1;
  st->fixed = fixed;
  if (st->may_slice()) st->release(fixed);              // ranges that end at a fixed frame: no clamp to the length
  return 0;
}

// rms: the frames not fed yet, which need the recording's end (their windows reach into the zero padding)
int slicer_finish(some_slicer_stream* st, const float* rms, int64_t n, int64_t n_samples) {
  SOME_REQUIRE(!st->finished, "some_slicer_stream_finish: the stream has finished");
  SOME_REQUIRE(n_samples >= st->fixed, "some_slicer_stream_finish: %lld samples, %lld were fixed already", (long long)n_samples,
               (long long)st->fixed);
  st->out.clear();
  st->fixed = n_samples;
  st->finished = true;
  if (st->core.feed(rms, n, st->queued)) return -1;
  const int64_t total = frames_whole(st->f, n_samples);
  if (total == 0) {                                       // one chunk
    st->queued.clear();
    st->out = {0, n_samples};
    return 0;
  }
  SOME_REQUIRE(st->core.known() == total, "some_slicer_stream_finish: %lld of the %lld frames of %lld samples were fed",
               (long long)st->core.known(), (long long)total, (long long)n_samples);
  if (st->core.finish(st->queued)) return -1;
  st->release(n_samples);
  return 0;
}
}  // namespace

extern "C" int some_slicer_stream_create(const some_slicer_frames* frames, some_slicer_stream** out) {
  SOME_REQUIRE(frames != nullptr && out != nullptr, "some_slicer_stream_create: null pointer");
  SOME_REQUIRE(frames->hop_size >= 1 && frames->win_size >= 1 && frames->max_sil_kept >= 1 && frames->min_interval >= 0 &&
                   frames->min_length >= 0,
               "some_slicer_stream_create: bad frame counts");
  *out = new some_slicer_stream(*frames);
  return 0;
}
extern "C" int some_slicer_stream_destroy(some_slicer_stream* st) {
  delete st;
  return 0;
}
extern "C" int some_slicer_stream_feed(some_slicer_stream* st, const float* rms, int n_frames, long long fixed,
                                       const int64_t** ranges, int* count) {
  SOME_REQUIRE(st != nullptr && (rms != nullptr || n_frames == 0) && n_frames >= 0 && ranges != nullptr && count != nullptr,
               "some_slicer_stream_feed: bad arguments");
  if (slicer_feed(st, rms, n_frames, fixed)) return -1;
  *ranges = st->out.data(), *count = static_cast<int>(st->out.size() / 2);
  return 0;
}
extern "C" int some_slicer_stream_finish(some_slicer_stream* st, const float* rms, int n_frames, long long n_samples,
                                         const int64_t** ranges, int* count) {
  SOME_REQUIRE(st != nullptr && (rms != nullptr || n_frames == 0) && n_frames >= 0 && ranges != nullptr && count != nullptr,
               "some_slicer_stream_finish: bad arguments");
  if (slicer_finish(st, rms, n_frames, n_samples)) return -1;
  *ranges = st->out.data(), *count = static_cast<int>(st->out.size() / 2);
  return 0;
}
extern "C" int some_slicer_stream_keep_from(const some_slicer_stream* st, long long* sample, long long* head,
                                            long long* rms_held) {
  SOME_REQUIRE(st != nullptr && sample != nullptr, "some_slicer_stream_keep_from: bad arguments");
  *sample = st->keep_from();
  if (head) *head = st->head();
  if (rms_held) *rms_held = static_cast<long long>(st->core.held());
  return 0;
}
