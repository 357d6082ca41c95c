// Native inference session: a model file written by `python -m some_b200.export` in, notes out, with no Python or torch in
// between.  Host code, and the copy kernel that scatters a stream step's upload; the work is done by the sm_90a kernels of
// this library, enqueued in the order Engine.enqueue (some_b200/engine.py) and Engine.infer_sliced use:
//   [some_resample_kaiser_windows] -> [some_slicer_rms_windows + the slicer's decisions on the host] -> per pipeline chunk:
//   some_mel_logmel -> some_forward (stand-alone LayerNorms, sigmoid / softmax head) -> some_decode_notes.
// The sliced and the encoded calls share that front end (Recordings: one resampling window per recording at another rate,
// one RMS window per recording that is cut, one batch over the chunks of all recordings); a stream step launches the same
// two kernels over the windows of its streams (both through StepWindows).  The encoded files call and the encoded stream
// step share the stage in front of it (Decode: one upload of the audio bytes, one FLAC scan, one PCM and one FLAC decode).
// A session holds one replica of the model per device it was opened on: the front end runs on replica 0, run_chunks spreads
// the chunks of each step over the replicas, each on its own thread (replica 0, the only one of a one-device session, on the
// calling thread), and take_chunks reads each caller's notes from the replica that ran each chunk.  Every call is a request in
// the session's queue (submit, at the end): calls of one kind that queue while a step runs share the next step, whose back
// end (run_chunks, Recordings, streams_step, bytes_step, peeks_step) takes the items of all of them.
//
// The model file (little-endian; INTEGRATION.md "Deploying without Python" has the table):
//   header     128 bytes: magic "SOMEB200", format version, ABI number, file size, directory offset, tensor count, the scalars
//              of the model (lay, outdim, quantized, sample rate, hop, win, midi_min, midi_max, midi_prob_deviation,
//              rest_threshold, bias correction applied) and the offset of the data section
//   directory  128 bytes per tensor: name (NUL-padded, 64 bytes), dtype, ndim, shape[4], offset, byte length
//   data       every tensor at a 256-byte aligned offset; the data section is uploaded as one block
// The whole file is read and validated before any CUDA call.
#include "host_common.h"

#include <limits.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../include/some_b200.h"
#include "audio_walk.h"

using namespace some;

namespace {

constexpr char kMagic[8] = {'S', 'O', 'M', 'E', 'B', '2', '0', '0'};
constexpr uint32_t kFormat = 1;
constexpr uint64_t kHeaderBytes = 128, kEntryBytes = 128, kAlign = 256;
constexpr int kNameBytes = 64;
enum { DT_F32 = 1, DT_BF16 = 2, DT_I32 = 3, DT_F64 = 4 };
constexpr int kKaiserTaps = 32769;   // resampy kaiser_best: 64 zero crossings x 512 + 1

// Engine's pipeline split (engine.py CHUNK_FRACTIONS / MIN_CHUNK_FRAMES): a small first chunk gets the GPU going while the
// next chunk is staged and copied.
constexpr double kChunkFractions[2] = {0.125, 0.375};
constexpr int kMinChunkFrames = 16384;

template <class T>
T rd(const uint8_t* p) {
  T v;
  memcpy(&v, p, sizeof(T));
  return v;
}

int dtype_bytes(uint32_t dt) { return dt == DT_F32 || dt == DT_I32 ? 4 : dt == DT_BF16 ? 2 : dt == DT_F64 ? 8 : 0; }
const char* dtype_name(uint32_t dt) {
  return dt == DT_F32 ? "f32" : dt == DT_BF16 ? "bf16" : dt == DT_I32 ? "i32" : dt == DT_F64 ? "f64" : "?";
}

// A tensor of the model file and the device pointer field it sets: at byte `field` of some_block_weights `block`, or of
// some_model when block < 0 (field < 0: the tensor is read by name).  A table row of count n > 1 is an array field, its
// tensors name.0 .. name.{n-1}; rows of one count next to each other go index-major (ln_g.0, ln_b.0, ln_g.1, ...).
struct Spec {
  std::string name;
  uint32_t dtype;
  std::vector<uint64_t> shape;
  ptrdiff_t field = -1;
  int count = 1, block = -1;
};

// A pointer field's offset and its count, from the field itself: 1, or the length of an array of pointers.
template <class F>
constexpr int pointer_count() {
  static_assert(std::is_pointer<typename std::remove_extent<F>::type>::value, "a tensor binds a pointer field");
  return static_cast<int>(sizeof(F) / sizeof(void*));
}
#define FIELD(S, f) static_cast<ptrdiff_t>(offsetof(S, f)), pointer_count<decltype(S::f)>()
#define BLOCK_FIELD(f) FIELD(some_block_weights, f)
#define MODEL_FIELD(f) FIELD(some_model, f)
#define BLOCK_FIELD32(f) FIELD(some_block_weights_f32, f)
#define MODEL_FIELD32(f) FIELD(some_model_f32, f)
constexpr uint64_t kDim = SOME_DIM, kFfn = 4 * SOME_DIM;
// The tensors of one block, under "blk<j>." (some_b200/weights.py: BLOCK_TENSORS).
const Spec kBlockRows[] = {
    {"ln_g", DT_F32, {kDim}, BLOCK_FIELD(ln_g)}, {"ln_b", DT_F32, {kDim}, BLOCK_FIELD(ln_b)},
    {"ffn_w1", DT_BF16, {kFfn, kDim}, BLOCK_FIELD(ffn_w1)}, {"ffn_b1", DT_F32, {kFfn}, BLOCK_FIELD(ffn_b1)},
    {"ffn_w2", DT_BF16, {kDim, kFfn}, BLOCK_FIELD(ffn_w2)}, {"ffn_b2", DT_F32, {kDim}, BLOCK_FIELD(ffn_b2)},
    {"w_qkv", DT_BF16, {3 * kDim, kDim}, BLOCK_FIELD(w_qkv)},
    {"w_out", DT_BF16, {kDim, kDim}, BLOCK_FIELD(w_out)}, {"b_out", DT_F32, {kDim}, BLOCK_FIELD(b_out)},
    {"w_pw1", DT_BF16, {2 * kDim, kDim}, BLOCK_FIELD(w_pw1)}, {"b_pw1", DT_F32, {2 * kDim}, BLOCK_FIELD(b_pw1)},
    {"w_dw", DT_F32, {SOME_CONV_K, kDim}, BLOCK_FIELD(w_dw)}, {"b_dw", DT_F32, {kDim}, BLOCK_FIELD(b_dw)},
    {"w_pw2", DT_BF16, {kDim, kDim}, BLOCK_FIELD(w_pw2)}, {"b_pw2", DT_F32, {kDim}, BLOCK_FIELD(b_pw2)}};
const Spec kInputRows[] = {{"w_in", DT_BF16, {kDim, SOME_N_MELS}, MODEL_FIELD(w_in)}, {"b_in", DT_F32, {kDim}, MODEL_FIELD(b_in)}};
const Spec kGluRows[] = {{"w", DT_BF16, {2 * kDim, kDim}}, {"b", DT_F32, {2 * kDim}}};     // under "glu<j>."
// The fp32 file's tensors (some_b200/weights.py: model_tensors_f32): the same names, order and shapes, every one f32 and bound
// into some_model_f32 / some_block_weights_f32; b_head is not padded.
const Spec kBlockRowsF32[] = {
    {"ln_g", DT_F32, {kDim}, BLOCK_FIELD32(ln_g)}, {"ln_b", DT_F32, {kDim}, BLOCK_FIELD32(ln_b)},
    {"ffn_w1", DT_F32, {kFfn, kDim}, BLOCK_FIELD32(ffn_w1)}, {"ffn_b1", DT_F32, {kFfn}, BLOCK_FIELD32(ffn_b1)},
    {"ffn_w2", DT_F32, {kDim, kFfn}, BLOCK_FIELD32(ffn_w2)}, {"ffn_b2", DT_F32, {kDim}, BLOCK_FIELD32(ffn_b2)},
    {"w_qkv", DT_F32, {3 * kDim, kDim}, BLOCK_FIELD32(w_qkv)},
    {"w_out", DT_F32, {kDim, kDim}, BLOCK_FIELD32(w_out)}, {"b_out", DT_F32, {kDim}, BLOCK_FIELD32(b_out)},
    {"w_pw1", DT_F32, {2 * kDim, kDim}, BLOCK_FIELD32(w_pw1)}, {"b_pw1", DT_F32, {2 * kDim}, BLOCK_FIELD32(b_pw1)},
    {"w_dw", DT_F32, {SOME_CONV_K, kDim}, BLOCK_FIELD32(w_dw)}, {"b_dw", DT_F32, {kDim}, BLOCK_FIELD32(b_dw)},
    {"w_pw2", DT_F32, {kDim, kDim}, BLOCK_FIELD32(w_pw2)}, {"b_pw2", DT_F32, {kDim}, BLOCK_FIELD32(b_pw2)}};
const Spec kInputRowsF32[] = {{"w_in", DT_F32, {kDim, SOME_N_MELS}, MODEL_FIELD32(w_in)},
                              {"b_in", DT_F32, {kDim}, MODEL_FIELD32(b_in)}};
const Spec kGluRowsF32[] = {{"w", DT_F32, {2 * kDim, kDim}}, {"b", DT_F32, {2 * kDim}}};

template <size_t n>
void add_rows(std::vector<Spec>& v, const std::string& prefix, int block, const Spec (&rows)[n]) {
  for (size_t i = 0, end; i < n; i = end) {
    for (end = i; end < n && rows[end].count == rows[i].count;) ++end;
    for (int k = 0; k < rows[i].count; ++k)
      for (size_t r = i; r < end; ++r) {
        Spec s = rows[r];
        if (s.count > 1) s.name += "." + std::to_string(k), s.field += k * static_cast<ptrdiff_t>(sizeof(void*));
        s.name = prefix + s.name, s.count = 1, s.block = block;
        v.push_back(s);
      }
  }
}

// The tensors a file of this geometry and precision must hold, in file order (some_b200/export.py: tensor_specs writes the
// same list).
std::vector<Spec> expected_tensors(int lay, int outdim, int precision) {
  const bool f32 = precision == SOME_PRECISION_FP32;
  const uint64_t n = static_cast<uint64_t>(outdim), n32 = static_cast<uint64_t>((outdim + 31) / 32 * 32);
  const Spec front[] = {
      {"mel_start", DT_I32, {SOME_N_MELS}}, {"mel_count", DT_I32, {SOME_N_MELS}},
      {"mel_weights", DT_F32, {SOME_N_MELS, SOME_MEL_MAXW}}, {"twiddle", DT_F32, {SOME_MEL_TW, 2}},
      {"window", DT_F32, {SOME_N_FFT}}, {"kaiser_best", DT_F64, {kKaiserTaps}}};
  const Spec head[] = {{"w_head", DT_BF16, {n, kDim}, MODEL_FIELD(w_head)}, {"b_head", DT_F32, {n32}, MODEL_FIELD(b_head)},
                       {"w_cut", DT_F32, {kDim}, MODEL_FIELD(w_cut)}, {"b_cut", DT_F32, {1}}};
  const Spec head32[] = {{"w_head", DT_F32, {n, kDim}, MODEL_FIELD32(w_head)}, {"b_head", DT_F32, {n}, MODEL_FIELD32(b_head)},
                         {"w_cut", DT_F32, {kDim}, MODEL_FIELD32(w_cut)}, {"b_cut", DT_F32, {1}}};
  std::vector<Spec> v;
  if (f32) add_rows(v, "", -1, kInputRowsF32);
  else add_rows(v, "", -1, kInputRows);
  for (int j = 0; j < 2 * (lay + 1); ++j) {
    if (f32) add_rows(v, "blk" + std::to_string(j) + ".", j, kBlockRowsF32);
    else add_rows(v, "blk" + std::to_string(j) + ".", j, kBlockRows);
  }
  for (int j = 0; j < 2 * lay; ++j) {
    if (f32) add_rows(v, "glu" + std::to_string(j) + ".", -1, kGluRowsF32);
    else add_rows(v, "glu" + std::to_string(j) + ".", -1, kGluRows);
  }
  if (f32) add_rows(v, "", -1, head32);
  else add_rows(v, "", -1, head);
  add_rows(v, "", -1, front);
  return v;
}

std::string shape_str(const std::vector<uint64_t>& s) {
  std::string r = "[";
  for (size_t i = 0; i < s.size(); ++i) r += (i ? ", " : "") + std::to_string(s[i]);
  return r + "]";
}

// A grow-only buffer of device memory, or of pinned host memory.  It frees itself, so the structs that own buffers need not
// list them; it is move-only, so a buffer has one owner.
template <bool kPinned>
struct GrowBuf {
  void* p = nullptr;
  size_t cap = 0;
  GrowBuf() = default;
  GrowBuf(GrowBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr, o.cap = 0; }
  GrowBuf& operator=(GrowBuf&& o) noexcept {
    release();
    p = o.p, cap = o.cap;
    o.p = nullptr, o.cap = 0;
    return *this;
  }
  ~GrowBuf() { release(); }
  int ensure(size_t bytes, const char* what) {
    if (bytes <= cap) return 0;
    const size_t want = std::max(bytes, cap + cap / 4);
    release();
    cudaError_t e = kPinned ? cudaHostAlloc(&p, want, cudaHostAllocDefault) : cudaMalloc(&p, want);
    SOME_REQUIRE(e == cudaSuccess, "session: %s(%zu) for %s: %s", kPinned ? "cudaHostAlloc" : "cudaMalloc", want, what,
                 cudaGetErrorString(e));
    cap = want;
    return 0;
  }
  void release() {
    if (p) kPinned ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr, cap = 0;
  }
};
using DevBuf = GrowBuf<false>;
using PinBuf = GrowBuf<true>;

// Makes `dev` current for the scope of a call and restores the caller's device afterwards.
struct DeviceScope {
  int prev = -1;
  cudaError_t err;
  explicit DeviceScope(int dev) {
    cudaGetDevice(&prev);
    err = cudaSetDevice(dev);
  }
  ~DeviceScope() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

#define SOME_CUDA(call, what)                                                           \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    SOME_REQUIRE(e_ == cudaSuccess, "session: %s: %s", what, cudaGetErrorString(e_));   \
  } while (0)

// n floats rounded up to a 16-byte multiple: where the next clip or recording of a buffer starts.
constexpr int64_t align4(int64_t n) { return (n + 3) & ~int64_t(3); }

struct Chunk {
  int c0, c1;
  uint64_t off;
  int bc, mc;
};

// A fixed set of worker threads for the host copies (staging of clips and recordings into pinned memory), kept for the
// session's lifetime like Engine._pool, so that no call creates threads.  run(n, fn) runs fn(0 .. n-1), lane 0 on the calling
// thread, and returns when every lane has finished; one step of the session runs at a time.
class WorkerPool {
 public:
  explicit WorkerPool(int n) : size_(std::max(1, n)) {
    for (int lane = 1; lane < size_; ++lane) threads_.emplace_back([this, lane] { loop(lane); });
  }
  ~WorkerPool() {
    {
      std::lock_guard<std::mutex> l(mu_);
      stop_ = true;
      ++gen_;
    }
    wake_.notify_all();
    for (auto& t : threads_) t.join();
  }
  int size() const { return size_; }
  void run(int n, const std::function<void(int)>& fn) {
    n = std::min(n, size_);
    if (n <= 1) {
      if (n == 1) fn(0);
      return;
    }
    {
      std::lock_guard<std::mutex> l(mu_);
      fn_ = &fn, lanes_ = n, pending_ = n - 1;
      ++gen_;
    }
    wake_.notify_all();
    fn(0);
    std::unique_lock<std::mutex> l(mu_);
    done_.wait(l, [this] { return pending_ == 0; });
    fn_ = nullptr;
  }

 private:
  void loop(int lane) {
    uint64_t seen = 0;
    for (;;) {
      const std::function<void(int)>* fn = nullptr;
      {
        std::unique_lock<std::mutex> l(mu_);
        wake_.wait(l, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
        if (lane >= lanes_) continue;        // not needed for this job
        fn = fn_;
      }
      (*fn)(lane);
      std::lock_guard<std::mutex> l(mu_);
      if (--pending_ == 0) done_.notify_one();
    }
  }
  int size_;
  std::vector<std::thread> threads_;
  std::mutex mu_;
  std::condition_variable wake_, done_;
  uint64_t gen_ = 0;
  bool stop_ = false;
  int lanes_ = 0, pending_ = 0;
  const std::function<void(int)>* fn_ = nullptr;
};

}  // namespace

struct some_notes {
  std::vector<int64_t> first;   // [clips + 1] prefix sums of the note counts
  std::vector<int64_t> range;   // [2 clips] sample range of each clip (sliced: in the resampled recording)
  std::vector<float> midi;
  std::vector<int32_t> dur;
  std::vector<uint8_t> rest;
  // the frame curves (some_notes_set_frames): `frames` asks for them, `framed` says the last fill wrote them
  bool frames = false, framed = false;
  std::vector<int64_t> frame_first;   // [clips + 1] prefix sums of the frame counts
  std::vector<float> f_midi, f_bound;
  std::vector<uint8_t> f_rest;
  std::vector<int32_t> f_note;
};

namespace {
struct Request;
// One copy of the model on one device, and what it needs to run a batch of chunks there: a session holds one replica per
// device it was opened on (a device listed twice holds two).  Replica 0 also runs the front end of every call.
struct Replica {
  int device = 0;
  void* weights = nullptr;
  std::vector<some_block_weights> blocks;
  std::vector<const uint16_t*> glu_w;
  std::vector<const float*> glu_b;
  some_model model{};
  // an fp32 file's model (some_session_get_precision): bound instead of `model`, run by some_forward_f32_tiled
  std::vector<some_block_weights_f32> blocks32;
  std::vector<const float*> glu_w32;
  some_model_f32 model32{};
  const int32_t *mel_start = nullptr, *mel_count = nullptr;
  const float *mel_weights = nullptr, *twiddle = nullptr, *window = nullptr;
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  cudaEvent_t ev[4] = {};
  // grow-only buffers of its batches; wave: the staged clips, or the chunks copied from replica 0's device
  DevBuf ws_block, scratch, wave_d, tab_d, cu_d, slab_d;
  PinBuf wave_h, tab_h, cu_h, slab_h;
  int ws_m = 0;
  some_workspace ws{};
  some_workspace_f32 ws32{};
  std::unique_ptr<WorkerPool> pool;       // its staging lanes (WorkerPool::run is not re-entrant)
  some_notes part;                        // the notes of its share of the step's chunks, in its order (no ranges)
  int64_t chunks = 0, frames = 0;         // its share of the step in progress
};
}  // namespace

struct some_session {
  // the calls waiting for a step (oldest first), whether a thread is running one, and the totals of some_session_get_stats,
  // all under mu; a caller waits on `done` until its own call has run
  mutable std::mutex mu;
  std::condition_variable done;
  std::deque<Request*> queue;
  bool running = false;
  some_session_stats stats{};
  some_session_info info{};
  int precision = SOME_PRECISION_BF16;
  float vmin = 0.f, vmax = 0.f, deviation = 1.f, threshold = 0.1f;
  std::vector<double> kaiser;             // host copy of the float64 table (scaled per rate pair on upload)
  // the device tables by downsampling ratio (1.0: the unscaled table every upsampling pair shares), each kept with the host
  // copy its upload reads
  struct Table {
    DevBuf d;
    std::vector<double> h;
  };
  std::map<double, Table> tables;
  // replica 0's device, stream and staging lanes, which the front end (uploads, decode, resampling, RMS) runs on
  int device = 0;
  cudaStream_t stream = nullptr;
  WorkerPool* pool = nullptr;
  // grow-only buffers on replica 0's device; rec_d: recordings at their own rates and at the model's (the sliced and
  // encoded calls)
  DevBuf rec_d, rms_d, step_d;
  PinBuf rms_h, step_h;                   // step: the samples and descriptors of a step's upload
  // the encoded calls' Decode: the audio bytes, the FLAC candidate list, scan workspace and int32 scratch
  DevBuf enc_d, flac_frames_d, flac_ws_d, flac_scratch_d;
  PinBuf enc_h, flac_frames_h;
  DevBuf peer_d;                          // the packed copies of a step's device audio that lies on other devices
  std::vector<std::unique_ptr<Replica>> reps;
  // lane r runs replica r's share of a step (lane 0 on the calling thread, the only lane of a one-device session); with
  // several replicas, `fed` is recorded on replica 0's stream once the front end has written the chunks the others copy
  std::unique_ptr<WorkerPool> lanes;
  cudaEvent_t fed = nullptr;
  std::vector<std::pair<int, int>> held;  // chunk c of the step: the replica that ran it, and its clip in that replica's part
  std::vector<std::pair<int64_t, int64_t>> load;   // each replica's chunks and frames in the last completed step
  bool frames = false;                    // the step in progress decodes frame curves (a result of it asks for them)
};

namespace {

void destroy(some_session* s) {
  s->lanes.reset();                       // joins the replicas' threads
  for (std::unique_ptr<Replica>& r : s->reps) {
    if (!r) continue;
    DeviceScope scope(r->device);
    if (r->stream) cudaStreamSynchronize(r->stream);
    if (r->copy_stream) cudaStreamSynchronize(r->copy_stream);
    for (cudaEvent_t& e : r->ev)
      if (e) cudaEventDestroy(e);
    if (r->stream) cudaStreamDestroy(r->stream);
    if (r->copy_stream) cudaStreamDestroy(r->copy_stream);
    if (r->weights) cudaFree(r->weights);
    r.reset();                            // its buffers free themselves, on its device
  }
  DeviceScope scope(s->device);
  if (s->fed) cudaEventDestroy(s->fed);
  delete s;                               // its buffers free themselves, on replica 0's device
}

// Empties *out for its next fill, which writes frame curves if it asks for them.
void clear(some_notes* out) {
  out->first.assign(1, 0), out->range.clear(), out->midi.clear(), out->dur.clear(), out->rest.clear();
  out->framed = out->frames;
  out->frame_first.assign(1, 0), out->f_midi.clear(), out->f_bound.clear(), out->f_rest.clear(), out->f_note.clear();
}

template <class T>
void append_range(std::vector<T>& to, const std::vector<T>& from, int64_t a, int64_t b) {
  to.insert(to.end(), from.begin() + a, from.begin() + b);
}

// Appends the notes of clip k of `from` to *out, as its next clip of sample range [b, e), and its frame curves when *out
// takes them (`from` then holds them: a step decodes curves when any of its results asks for them).
void append_clip(const some_notes& from, int k, int64_t b, int64_t e, some_notes* out) {
  const int64_t n0 = from.first[k], n1 = from.first[k + 1];
  append_range(out->midi, from.midi, n0, n1);
  append_range(out->dur, from.dur, n0, n1);
  append_range(out->rest, from.rest, n0, n1);
  out->first.push_back(out->first.back() + (n1 - n0));
  out->range.push_back(b), out->range.push_back(e);
  if (!out->framed) return;
  const int64_t f0 = from.frame_first[k], f1 = from.frame_first[k + 1];
  append_range(out->f_midi, from.f_midi, f0, f1);
  append_range(out->f_bound, from.f_bound, f0, f1);
  append_range(out->f_rest, from.f_rest, f0, f1);
  append_range(out->f_note, from.f_note, f0, f1);
  out->frame_first.push_back(out->frame_first.back() + (f1 - f0));
}

// Sets *out to chunks [c0, c1) of the step's last run_chunks, each read from the replica that ran it, with their frame curves
// when *out asks for them; chunk c is samples [begin[c], begin[c] + lens[c]).
void take_chunks(const some_session* s, int c0, int c1, const int64_t* begin, const int64_t* lens, some_notes* out) {
  clear(out);
  for (int c = c0; c < c1; ++c)
    append_clip(s->reps[s->held[c].first]->part, s->held[c].second, begin[c], begin[c] + lens[c], out);
}

// A span of host memory to copy into pinned memory.
struct HostSpan {
  void* dst;
  const void* src;
  size_t bytes;
};
// Copies the spans on the session's threads: each span in pieces of up to `piece` bytes, dealt out in turn to one thread per
// `piece` bytes in all (at most the pool's size).
void copy_to_pinned(WorkerPool& pool, const std::vector<HostSpan>& spans, size_t piece) {
  std::vector<std::pair<const HostSpan*, size_t>> pieces;
  size_t total = 0;
  for (const HostSpan& sp : spans) {
    for (size_t a = 0; a < sp.bytes; a += piece) pieces.push_back({&sp, a});
    total += sp.bytes;
  }
  const int nt = static_cast<int>(std::min<size_t>(pool.size(), (total + piece - 1) / piece));
  pool.run(nt, [&](int t) {
    for (size_t j = t; j < pieces.size(); j += nt) {
      const HostSpan& sp = *pieces[j].first;
      const size_t a = pieces[j].second;
      memcpy(static_cast<char*>(sp.dst) + a, static_cast<const char*>(sp.src) + a, std::min(piece, sp.bytes - a));
    }
  });
}

// Engine._chunks: up to three pipeline chunks of whole clips, a small first one.
std::vector<std::pair<int, int>> split_chunks(const std::vector<int32_t>& cu) {
  const int b = static_cast<int>(cu.size()) - 1;
  const int64_t m = cu[b];
  if (b < 2 || m < 2 * kMinChunkFrames) return {{0, b}};
  std::vector<int> bounds{0};
  double acc = 0.0;
  for (double f : kChunkFractions) {
    acc += f;
    const double target = acc * static_cast<double>(m);
    int i = static_cast<int>(std::lower_bound(cu.begin(), cu.end(), target,
                                              [](int32_t v, double t) { return static_cast<double>(v) < t; }) -
                             cu.begin());
    i = std::min(std::max(i, bounds.back() + 1), b - 1);
    if (cu[i] - cu[bounds.back()] >= kMinChunkFrames / 2 && i > bounds.back()) bounds.push_back(i);
  }
  bounds.push_back(b);
  std::vector<std::pair<int, int>> out;
  for (size_t i = 0; i + 1 < bounds.size(); ++i)
    if (bounds[i + 1] > bounds[i]) out.push_back({bounds[i], bounds[i + 1]});
  return out;
}

// One var-len batch through mel -> trunk -> decode on replica r, pipelined like Engine.enqueue.  Host clips (`host` != NULL:
// clip i is host[i][0 .. lens[i])) are staged through pinned memory and copied on the copy stream while the previous chunk's
// kernels run; resident clips (`resident` != NULL) are the sample ranges [starts[i], starts[i] + lens[i]) of that buffer on
// r's device, written by work on r's streams or awaited by its copy stream.  The notes of clip i go to clip i of r.part.
//   Each pipeline chunk's results come down in one slab, one copy for the whole batch.  Per chunk of bc clips and mc frames:
// note counts i32 [bc] | durations i32 [mc] | MIDI f32 [mc] | rests u8 [mc], padded to 16 bytes.  When the step decodes
// frame curves (s->frames), the chunk's region goes on with its curves, padded to 16 bytes: the decode's per-frame values
// f32 [mc], the bounds f32 [mc] (a device copy of the trunk's output, so the slab still comes down in one copy), the frame ->
// note index i32 [mc] and the rest flags u8 [mc], 13 bytes per frame.  A step without curves copies what it copied before.
int run_batch(const some_session* s, Replica& r, const float* const* host, const float* resident, const int64_t* res_starts,
              const int64_t* lens, int B) {
  std::vector<int32_t> cu(B + 1, 0);
  std::vector<int64_t> starts(B, 0);
  int64_t total = 0;
  for (int i = 0; i < B; ++i) {
    SOME_REQUIRE(lens[i] >= 0, "session: clip %d has a negative length", i);
    const int64_t frames = 1 + lens[i] / SOME_HOP;
    SOME_REQUIRE(cu[i] + frames < (int64_t(1) << 31), "session: the batch has more than 2^31 frames");
    cu[i + 1] = static_cast<int32_t>(cu[i] + frames);
    if (host) {
      starts[i] = total;
      total += align4(lens[i]);                 // 16-byte aligned clip starts, as Engine.tables
    } else {
      starts[i] = res_starts[i];
    }
  }
  const auto spans = split_chunks(cu);
  std::vector<Chunk> layout;
  uint64_t slab_bytes = 0;
  int max_mc = 1;
  auto notes_bytes = [](const Chunk& ch) { return (4ull * ch.bc + 9ull * ch.mc + 15) & ~uint64_t(15); };
  for (const auto& sp : spans) {
    const int bc = sp.second - sp.first, mc = cu[sp.second] - cu[sp.first];
    layout.push_back({sp.first, sp.second, slab_bytes, bc, mc});
    slab_bytes += notes_bytes(layout.back());
    if (s->frames) slab_bytes += (13ull * mc + 15) & ~uint64_t(15);
    max_mc = std::max(max_mc, mc);
  }
  // buffers
  const bool f32 = s->precision == SOME_PRECISION_FP32;
  if (max_mc > r.ws_m) {
    const uint64_t bytes = f32 ? some_workspace_f32_bytes(max_mc, s->info.outdim) : some_workspace_bytes(max_mc, s->info.outdim, 0);
    if (r.ws_block.ensure(bytes, "the workspace")) return -1;
    if (f32 ? some_workspace_f32_carve(r.ws_block.p, r.ws_block.cap, max_mc, s->info.outdim, &r.ws32)
            : some_workspace_carve(r.ws_block.p, r.ws_block.cap, max_mc, s->info.outdim, 0, &r.ws))
      return -1;
    if (r.scratch.ensure(some_decode_scratch_bytes(max_mc), "the decode scratch")) return -1;
    r.ws_m = max_mc;
  }
  if (r.tab_h.ensure(16ull * B + 16, "tables") || r.tab_d.ensure(16ull * B + 16, "tables") ||
      r.cu_h.ensure(4ull * (B + layout.size()) + 4, "cu_frames") || r.cu_d.ensure(4ull * (B + layout.size()) + 4, "cu_frames") ||
      r.slab_h.ensure(slab_bytes + 16, "the note slab") || r.slab_d.ensure(slab_bytes + 16, "the note slab"))
    return -1;
  if (host && (r.wave_h.ensure(4ull * total + 16, "the staged audio") || r.wave_d.ensure(4ull * total + 16, "the audio")))
    return -1;
  float* wave_h = static_cast<float*>(r.wave_h.p);
  const float* wave = host ? static_cast<const float*>(r.wave_d.p) : resident;
  int64_t* tab_h = static_cast<int64_t*>(r.tab_h.p);
  int64_t* tab_d = static_cast<int64_t*>(r.tab_d.p);
  int32_t* cu_h = static_cast<int32_t*>(r.cu_h.p);
  int32_t* cu_d = static_cast<int32_t*>(r.cu_d.p);
  uint8_t* slab = static_cast<uint8_t*>(r.slab_d.p);
  const int head = s->info.quantized ? SOME_EPI_SOFTMAX_F32 : SOME_EPI_SIGMOID_F32;
  const float* probs = f32 ? r.ws32.probs : r.ws.probs;
  const float* bounds = f32 ? r.ws32.bounds : r.ws.bounds;

  for (size_t ci = 0; ci < layout.size(); ++ci) {
    const Chunk& ch = layout[ci];
    const int64_t lo = starts[ch.c0];
    if (host) {                                  // stage this chunk's clips; the GPU is still busy with the previous chunk
      const int nt = std::min(r.pool->size(), ch.bc);
      r.pool->run(nt, [&](int t) {
        for (int i = ch.c0 + t; i < ch.c1; i += nt)
          if (lens[i]) memcpy(wave_h + starts[i], host[i], 4ull * lens[i]);
      });
    }
    int64_t* tab = tab_h + 2 * ch.c0;
    int max_frames = 1;
    for (int i = 0; i < ch.bc; ++i) {
      tab[i] = starts[ch.c0 + i] - lo;
      tab[ch.bc + i] = lens[ch.c0 + i];
      max_frames = std::max(max_frames, cu[ch.c0 + i + 1] - cu[ch.c0 + i]);
    }
    int32_t* cuc = cu_h + ch.c0 + ci;            // chunk ci owns entries [c0 + ci, c1 + ci]
    for (int i = 0; i <= ch.bc; ++i) cuc[i] = cu[ch.c0 + i] - cu[ch.c0];
    const int64_t hi = host ? starts[ch.c1 - 1] + align4(lens[ch.c1 - 1]) : lo;
    if (hi > lo)
      SOME_CUDA(cudaMemcpyAsync(static_cast<float*>(r.wave_d.p) + lo, wave_h + lo, 4ull * (hi - lo), cudaMemcpyHostToDevice,
                                r.copy_stream), "audio upload");
    SOME_CUDA(cudaMemcpyAsync(tab_d + 2 * ch.c0, tab, 16ull * ch.bc, cudaMemcpyHostToDevice, r.copy_stream), "table upload");
    SOME_CUDA(cudaMemcpyAsync(cu_d + ch.c0 + ci, cuc, 4ull * (ch.bc + 1), cudaMemcpyHostToDevice, r.copy_stream),
              "cu_frames upload");
    SOME_CUDA(cudaEventRecord(r.ev[ci], r.copy_stream), "event record");
    SOME_CUDA(cudaStreamWaitEvent(r.stream, r.ev[ci], 0), "stream wait");

    const int32_t* cud = cu_d + ch.c0 + ci;
    uint8_t* o = slab + ch.off;
    // an fp32 session writes the mel as f32 and runs the fp32 trunk (Engine.enqueue(..., precision='fp32'))
    if (some_mel_logmel(wave + lo, tab_d + 2 * ch.c0, tab_d + 2 * ch.c0 + ch.bc, cud, ch.bc, max_frames, r.mel_start,
                        r.mel_count, r.mel_weights, r.twiddle, r.window, f32 ? const_cast<float*>(r.ws32.units) : nullptr,
                        f32 ? nullptr : const_cast<uint16_t*>(r.ws.units), 1e-5f, r.stream))
      return -1;
    if (f32 ? some_forward_f32_tiled(&r.model32, &r.ws32, ch.mc, ch.bc, cud, max_frames, head, r.stream)
            : some_forward(&r.model, &r.ws, ch.mc, ch.bc, cud, max_frames, head, nullptr, nullptr, r.stream))
      return -1;
    some_decode_args d{};
    d.probs = probs, d.bounds = bounds, d.cu_frames = cud;
    d.B = ch.bc, d.M = ch.mc, d.N = s->info.outdim, d.quantized = s->info.quantized;
    d.vmin = s->vmin, d.vmax = s->vmax, d.deviation = s->deviation, d.threshold = s->threshold;
    d.note_count = reinterpret_cast<int32_t*>(o);
    d.note_dur = reinterpret_cast<int32_t*>(o + 4ull * ch.bc);
    d.note_midi = reinterpret_cast<float*>(o + 4ull * ch.bc + 4ull * ch.mc);
    d.note_rest = o + 4ull * ch.bc + 8ull * ch.mc;
    d.scratch = r.scratch.p;
    uint8_t* f = o + notes_bytes(ch);
    if (s->frames) {
      d.dbg_values = reinterpret_cast<float*>(f);
      d.dbg_frame2item = reinterpret_cast<int32_t*>(f + 8ull * ch.mc);
      d.dbg_rest = f + 12ull * ch.mc;
    }
    if (some_decode_notes(&d, r.stream)) return -1;
    if (s->frames)
      SOME_CUDA(cudaMemcpyAsync(f + 4ull * ch.mc, bounds, 4ull * ch.mc, cudaMemcpyDeviceToDevice, r.stream), "bounds copy");
  }
  if (slab_bytes) SOME_CUDA(cudaMemcpyAsync(r.slab_h.p, slab, slab_bytes, cudaMemcpyDeviceToHost, r.stream), "note download");
  SOME_CUDA(cudaStreamSynchronize(r.stream), "synchronise");

  // unpack: the notes of clip b start at its first frame's row of the chunk slab, and so do its curves
  some_notes* out = &r.part;
  out->frames = s->frames;
  clear(out);
  const uint8_t* h = static_cast<const uint8_t*>(r.slab_h.p);
  for (const Chunk& ch : layout) {
    const uint8_t* o = h + ch.off;
    for (int b = 0; b < ch.bc; ++b) {
      const int32_t n = rd<int32_t>(o + 4ull * b);
      const int64_t row = cu[ch.c0 + b] - cu[ch.c0];
      const int32_t T = cu[ch.c0 + b + 1] - cu[ch.c0 + b];
      SOME_REQUIRE(n >= 0 && row + n <= ch.mc, "session: decode returned %d notes for a clip of %d frames", n, T);
      for (int j = 0; j < n; ++j) {
        const uint64_t r = static_cast<uint64_t>(row + j);
        out->dur.push_back(rd<int32_t>(o + 4ull * ch.bc + 4 * r));
        out->midi.push_back(rd<float>(o + 4ull * ch.bc + 4ull * ch.mc + 4 * r));
        out->rest.push_back(o[4ull * ch.bc + 8ull * ch.mc + r]);
      }
      out->first.push_back(out->first.back() + n);
      if (!s->frames) continue;
      const uint8_t* f = o + notes_bytes(ch);
      auto put = [&](auto& to, const uint8_t* at) {
        using T_ = typename std::remove_reference<decltype(to)>::type::value_type;
        const size_t k = to.size();
        to.resize(k + T);
        memcpy(to.data() + k, at + sizeof(T_) * row, sizeof(T_) * T);
      };
      put(out->f_midi, f);
      put(out->f_bound, f + 4ull * ch.mc);
      put(out->f_note, f + 8ull * ch.mc);
      put(out->f_rest, f + 12ull * ch.mc);
      out->frame_first.push_back(out->frame_first.back() + T);
    }
  }
  return 0;
}

// The chunks of a step, on every replica of the session: some_shard_clips assigns them (one replica runs all of them);
// replica 0 runs its share on the calling thread and replica r > 0 its share on lane r, with the caller's some_set_pdl
// setting, each through run_batch into its own part, and s->held records which replica ran each chunk and where its notes
// lie there, for take_chunks (a chunk's notes do not depend on the rest of its batch).  Resident chunks lie in a buffer on
// replica 0's device, written on its stream: replica r > 0 waits on its copy stream for `fed`, recorded there after the
// front end, and copies its share, packed at 16-byte aligned starts, into its own audio buffer (a peer copy, or a
// device-to-device copy when both replicas are on one device).  Host clips are staged straight to the replica that runs them.
int run_chunks(some_session* s, const float* const* host, const float* resident, const int64_t* starts, const int64_t* lens,
               int B) {
  const int R = static_cast<int>(s->reps.size());
  std::vector<int32_t> owner(B, 0);
  if (R > 1 && some_shard_clips(lens, B, R, owner.data())) return -1;
  std::vector<std::vector<int>> share(R);
  s->held.resize(B);
  for (int c = 0; c < B; ++c) {
    s->held[c] = {owner[c], static_cast<int>(share[owner[c]].size())};
    share[owner[c]].push_back(c);
  }
  if (resident && std::any_of(share.begin() + 1, share.end(), [](const std::vector<int>& v) { return !v.empty(); }))
    SOME_CUDA(cudaEventRecord(s->fed, s->stream), "event record");
  const int pdl = pdl_enabled() ? 1 : 0;
  std::vector<int> rc(R, 0);
  std::vector<std::string> err(R);
  s->lanes->run(R, [&](int ri) {
    Replica& r = *s->reps[ri];
    const std::vector<int>& mine = share[ri];
    const int b = static_cast<int>(mine.size());
    if (b == 0) return;
    std::vector<const float*> clips;
    std::vector<int64_t> at, len;
    int64_t total = 0;
    for (int c : mine) {
      len.push_back(lens[c]);
      r.frames += 1 + lens[c] / SOME_HOP;
      if (host) clips.push_back(host[c]);
      else if (ri == 0) at.push_back(starts[c]);
      else at.push_back(total), total += align4(lens[c]);
    }
    r.chunks = b;
    auto work = [&]() -> int {
      if (!resident || ri == 0) return run_batch(s, r, host ? clips.data() : nullptr, resident, at.data(), len.data(), b);
      if (r.wave_d.ensure(4ull * total + 16, "the audio")) return -1;
      float* wave = static_cast<float*>(r.wave_d.p);
      SOME_CUDA(cudaStreamWaitEvent(r.copy_stream, s->fed, 0), "stream wait");
      for (int k = 0; k < b; ++k)
        if (len[k])
          SOME_CUDA(cudaMemcpyPeerAsync(wave + at[k], r.device, resident + starts[mine[k]], s->device, 4ull * len[k],
                                        r.copy_stream), "chunk copy");
      return run_batch(s, r, nullptr, wave, at.data(), len.data(), b);
    };
    if (ri == 0) {
      rc[ri] = work();
    } else {
      some_set_pdl(pdl);
      DeviceScope scope(r.device);
      if (scope.err != cudaSuccess) set_error("cudaSetDevice: %s", cudaGetErrorString(scope.err)), rc[ri] = -1;
      else rc[ri] = work();
    }
    if (rc[ri]) err[ri] = some_last_error();
  });
  for (int ri = 0; ri < R; ++ri)
    if (rc[ri]) {
      if (R > 1) set_error("device %d (replica %d): %s", s->reps[ri]->device, ri, err[ri].c_str());   // one replica: as is
      return -1;
    }
  return 0;
}

// Host floats to upload: n floats at src go to dst.
struct Staged {
  float* dst;
  const float* src;
  int64_t n;
};
// Uploads host recordings through the pinned staging buffer, each at its own place there: in pieces of 16 MB, each copied
// into pinned memory by the session's threads (256 KB per thread and turn) and then sent while the next piece is copied.
int upload_staged(some_session* s, const std::vector<Staged>& recs) {
  constexpr int64_t kPiece = int64_t(1) << 22;
  int64_t total = 0;
  for (const Staged& r : recs) total += align4(r.n);
  PinBuf& staging = s->reps[0]->wave_h;
  if (staging.ensure(4ull * total + 16, "the staged audio")) return -1;
  float* pin = static_cast<float*>(staging.p);
  for (const Staged& r : recs) {
    for (int64_t a = 0; a < r.n; a += kPiece) {
      const int64_t len = std::min(kPiece, r.n - a);
      copy_to_pinned(*s->pool, {{pin + a, r.src + a, 4ull * len}}, size_t(1) << 18);
      SOME_CUDA(cudaMemcpyAsync(r.dst + a, pin + a, 4ull * len, cudaMemcpyHostToDevice, s->stream), "audio upload");
    }
    pin += align4(r.n);
  }
  return 0;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------- results
extern "C" int some_notes_create(some_notes** out) {
  SOME_REQUIRE(out != nullptr, "some_notes_create: null pointer");
  *out = new some_notes();
  (*out)->first.assign(1, 0);
  return 0;
}
extern "C" int some_notes_destroy(some_notes* n) {
  delete n;
  return 0;
}
extern "C" int some_notes_clips(const some_notes* n) {
  SOME_REQUIRE(n != nullptr, "some_notes_clips: null pointer");
  return static_cast<int>(n->first.size()) - 1;
}
extern "C" int some_notes_get(const some_notes* n, int clip, int* count, const float** note_midi, const int32_t** note_dur,
                              const uint8_t** note_rest, int64_t* begin, int64_t* end) {
  SOME_REQUIRE(n != nullptr && clip >= 0 && clip + 1 < static_cast<int>(n->first.size()),
               "some_notes_get: clip %d out of range", clip);
  const int64_t a = n->first[clip];
  if (count) *count = static_cast<int>(n->first[clip + 1] - a);
  if (note_midi) *note_midi = n->midi.data() + a;
  if (note_dur) *note_dur = n->dur.data() + a;
  if (note_rest) *note_rest = n->rest.data() + a;
  if (begin) *begin = n->range[2 * clip];
  if (end) *end = n->range[2 * clip + 1];
  return 0;
}
extern "C" int some_notes_set_frames(some_notes* n, int on) {
  SOME_REQUIRE(n != nullptr, "some_notes_set_frames: null pointer");
  n->frames = on != 0;
  return 0;
}
extern "C" int some_notes_get_frames(const some_notes* n, int clip, int* frames, const float** midi, const uint8_t** rest,
                                     const float** bound, const int32_t** note_index) {
  SOME_REQUIRE(n != nullptr, "some_notes_get_frames: null pointer");
  SOME_REQUIRE(clip >= 0 && clip + 1 < static_cast<int>(n->first.size()), "some_notes_get_frames: clip %d out of range", clip);
  SOME_REQUIRE(n->framed, "some_notes_get_frames: the notes were filled with frames off (some_notes_set_frames)");
  const int64_t a = n->frame_first[clip];
  if (frames) *frames = static_cast<int>(n->frame_first[clip + 1] - a);
  if (midi) *midi = n->f_midi.data() + a;
  if (rest) *rest = n->f_rest.data() + a;
  if (bound) *bound = n->f_bound.data() + a;
  if (note_index) *note_index = n->f_note.data() + a;
  return 0;
}

// ---------------------------------------------------------------------------------------------------- session
namespace {
constexpr int kMaxReplicas = 64;

// Points a replica's model and mel tables into its copy of the weights; dp(name) is a tensor's device address there.
template <class Dp>
void bind_weights(Replica& r, const std::vector<Spec>& specs, int lay, int outdim, bool f32, Dp dp) {
  auto fl = [&](const std::string& n) { return static_cast<const float*>(dp(n)); };
  some_model& m = r.model;
  some_model_f32& m32 = r.model32;
  if (f32) r.blocks32.resize(2 * (lay + 1));
  else r.blocks.resize(2 * (lay + 1));       // value-initialised: the LayerNorm-folded fields stay null
  for (const Spec& sp : specs) {
    if (sp.field < 0) continue;
    const void* p = dp(sp.name);
    void* target = f32 ? (sp.block < 0 ? static_cast<void*>(&m32) : static_cast<void*>(&r.blocks32[sp.block]))
                       : (sp.block < 0 ? static_cast<void*>(&m) : static_cast<void*>(&r.blocks[sp.block]));
    memcpy(static_cast<uint8_t*>(target) + sp.field, &p, sizeof(p));
  }
  for (int j = 0; j < 2 * lay; ++j) {
    if (f32) r.glu_w32.push_back(fl("glu" + std::to_string(j) + ".w"));
    else r.glu_w.push_back(static_cast<const uint16_t*>(dp("glu" + std::to_string(j) + ".w")));
    r.glu_b.push_back(fl("glu" + std::to_string(j) + ".b"));
  }
  if (lay == 0) r.glu_w.push_back(nullptr), r.glu_w32.push_back(nullptr), r.glu_b.push_back(nullptr);
  if (f32) {
    m32.lay = lay, m32.outdim = outdim;
    m32.blocks = r.blocks32.data();
    m32.glu_w = r.glu_w32.data();
    m32.glu_b = r.glu_b.data();
  } else {
    m.lay = lay, m.outdim = outdim;
    m.blocks = r.blocks.data();
    m.glu_w = r.glu_w.data();
    m.glu_b = r.glu_b.data();
    m.ln_fold = 0;                                // the default stand-alone LayerNorm sequence
  }
  r.mel_start = static_cast<const int32_t*>(dp("mel_start"));
  r.mel_count = static_cast<const int32_t*>(dp("mel_count"));
  r.mel_weights = fl("mel_weights"), r.twiddle = fl("twiddle"), r.window = fl("window");
}

// some_session_open_devices, after its arguments are checked; `who` names the function in messages, and `listed` adds the
// index of a refused device in the list.
int open_session(const char* who, const char* path, const int* devices, int n, bool listed, some_session** out) {
  FILE* fp = fopen(path, "rb");
  SOME_REQUIRE(fp != nullptr, "%s: cannot open the model file", path);
  std::vector<uint8_t> file;
  {
    uint8_t buf[1 << 16];
    size_t got;
    while ((got = fread(buf, 1, sizeof(buf), fp)) > 0) file.insert(file.end(), buf, buf + got);
    const bool bad = ferror(fp) != 0;
    fclose(fp);
    SOME_REQUIRE(!bad, "%s: read error", path);
  }
  const uint64_t size = file.size();
  const uint8_t* f = file.data();
  // ---- header
  SOME_REQUIRE(size >= kHeaderBytes, "%s: truncated header (%llu bytes, a model file starts with %llu)", path,
               (unsigned long long)size, (unsigned long long)kHeaderBytes);
  SOME_REQUIRE(memcmp(f, kMagic, 8) == 0, "%s: bad magic: not a some_b200 model file", path);
  const uint32_t format = rd<uint32_t>(f + 8), abi = rd<uint32_t>(f + 12);
  SOME_REQUIRE(format == kFormat, "%s: unsupported format version %u (this library reads version %u)", path, format, kFormat);
  SOME_REQUIRE(abi == SOME_B200_VERSION, "%s: written for ABI %u, this library is ABI %d", path, abi, SOME_B200_VERSION);
  const uint64_t file_size = rd<uint64_t>(f + 16), dir_off = rd<uint64_t>(f + 24), data_off = rd<uint64_t>(f + 80);
  const uint32_t n_tensors = rd<uint32_t>(f + 32);
  const int32_t lay = rd<int32_t>(f + 36), outdim = rd<int32_t>(f + 40), quantized = rd<int32_t>(f + 44);
  const int32_t sr = rd<int32_t>(f + 48), hop = rd<int32_t>(f + 52), win = rd<int32_t>(f + 56);
  const int32_t bias_corrected = rd<int32_t>(f + 76);
  const int32_t precision = rd<int32_t>(f + 88);    // zero in bf16 files
  SOME_REQUIRE(dir_off >= kHeaderBytes && dir_off <= size && n_tensors <= (size - dir_off) / kEntryBytes,
               "%s: truncated directory (%u entries at byte %llu, file of %llu bytes)", path, n_tensors,
               (unsigned long long)dir_off, (unsigned long long)size);
  SOME_REQUIRE(file_size == size, "%s: file size %llu does not match the %llu bytes the header records", path,
               (unsigned long long)size, (unsigned long long)file_size);
  SOME_REQUIRE(data_off % kAlign == 0 && data_off >= dir_off + uint64_t(n_tensors) * kEntryBytes && data_off <= size,
               "%s: bad data offset %llu", path, (unsigned long long)data_off);
  SOME_REQUIRE(lay >= 0 && lay <= 64 && outdim >= 1 && outdim <= 256 && (quantized == 0 || quantized == 1) && sr > 0 &&
                   hop == SOME_HOP && win == SOME_N_FFT,
               "%s: unsupported model scalars (lay %d, outdim %d, quantized %d, rate %d, hop %d, win %d)", path, lay, outdim,
               quantized, sr, hop, win);
  SOME_REQUIRE(precision == SOME_PRECISION_BF16 || precision == SOME_PRECISION_FP32,
               "%s: unknown precision %d in the header (0 = bf16, 1 = fp32)", path, precision);
  // ---- directory
  struct Entry {
    uint32_t dtype;
    std::vector<uint64_t> shape;
    uint64_t off, bytes;
  };
  std::map<std::string, Entry> dir;
  for (uint32_t t = 0; t < n_tensors; ++t) {
    const uint8_t* e = f + dir_off + uint64_t(t) * kEntryBytes;
    char name[kNameBytes + 1] = {};
    memcpy(name, e, kNameBytes);
    Entry en;
    en.dtype = rd<uint32_t>(e + 64);
    const uint32_t ndim = rd<uint32_t>(e + 68);
    SOME_REQUIRE(ndim <= 4 && dtype_bytes(en.dtype) > 0, "%s: directory entry %u ('%s') has dtype %u / %u dimensions", path, t,
                 name, en.dtype, ndim);
    uint64_t elems = 1;
    for (uint32_t k = 0; k < ndim; ++k) {
      en.shape.push_back(rd<uint64_t>(e + 72 + 8 * k));
      SOME_REQUIRE(en.shape.back() < (uint64_t(1) << 40), "%s: tensor '%s' has an absurd shape", path, name);
      elems *= en.shape.back();
    }
    en.off = rd<uint64_t>(e + 104);
    en.bytes = rd<uint64_t>(e + 112);
    SOME_REQUIRE(en.off % kAlign == 0 && en.off >= data_off && en.off <= size && en.bytes <= size - en.off,
                 "%s: tensor '%s' lies outside the data section (bytes %llu + %llu of %llu)", path, name,
                 (unsigned long long)en.off, (unsigned long long)en.bytes, (unsigned long long)size);
    SOME_REQUIRE(en.bytes == elems * dtype_bytes(en.dtype), "%s: tensor '%s' holds %llu bytes, its shape needs %llu", path,
                 name, (unsigned long long)en.bytes, (unsigned long long)(elems * dtype_bytes(en.dtype)));
    SOME_REQUIRE(dir.emplace(name, en).second, "%s: tensor '%s' appears twice", path, name);
  }
  const std::vector<Spec> specs = expected_tensors(lay, outdim, precision);
  for (const Spec& sp : specs) {
    auto it = dir.find(sp.name);
    SOME_REQUIRE(it != dir.end(), "%s: missing tensor '%s'", path, sp.name.c_str());
    SOME_REQUIRE(it->second.dtype == sp.dtype && it->second.shape == sp.shape,
                 "%s: tensor '%s' is %s %s, a%s model with lay %d / outdim %d needs %s %s", path, sp.name.c_str(),
                 dtype_name(it->second.dtype), shape_str(it->second.shape).c_str(),
                 precision == SOME_PRECISION_FP32 ? "n fp32" : " bf16", lay, outdim, dtype_name(sp.dtype),
                 shape_str(sp.shape).c_str());
  }
  SOME_REQUIRE(dir.size() == specs.size(), "%s: %zu tensors, a model with lay %d / outdim %d has %zu", path, dir.size(), lay,
               outdim, specs.size());

  // ---- the devices (first CUDA call), every one checked before anything is allocated
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  for (int i = 0; i < n; ++i) {
    const int device = devices[i];
    char at[32] = "";
    if (listed) snprintf(at, sizeof(at), "devices[%d]: ", i);
    SOME_REQUIRE(e == cudaSuccess && device >= 0 && device < n_dev, "%s: %sno CUDA device %d (%s)", who, at, device,
                 e == cudaSuccess ? "out of range" : cudaGetErrorString(e));
    cudaDeviceProp prop;
    SOME_CUDA(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties");
    SOME_REQUIRE(prop.major == 9 && prop.minor == 0, "%s: %sdevice %d (%s) is sm_%d%d; the kernels are built for sm_90a", who,
                 at, device, prop.name, prop.major, prop.minor);
  }
  some_session* s = new some_session();
  s->device = devices[0];
  auto fail = [&](int rc) {
    destroy(s);
    return rc;
  };
  const unsigned hw = std::thread::hardware_concurrency();
  const int lanes = static_cast<int>(std::min(8u, std::max(2u, hw / 2)));
  for (int i = 0; i < n; ++i) {
    const int device = devices[i];
    char at[32] = "";
    if (listed) snprintf(at, sizeof(at), "devices[%d]: ", i);
    s->reps.emplace_back(new Replica());
    Replica& r = *s->reps.back();
    r.device = device;
    DeviceScope scope(device);
    if (scope.err != cudaSuccess) {
      set_error("%s: %scudaSetDevice(%d): %s", who, at, device, cudaGetErrorString(scope.err));
      return fail(-2);
    }
    e = cudaStreamCreateWithFlags(&r.stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&r.copy_stream, cudaStreamNonBlocking);
    for (cudaEvent_t& ev : r.ev)
      if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    // the weights go up on the replica's own (non-blocking) stream, which every later kernel of the replica runs on; the wait
    // also keeps the host copy of the file alive until the copy has read it
    if (e == cudaSuccess) e = cudaMalloc(&r.weights, std::max<uint64_t>(size - data_off, 1));
    if (e == cudaSuccess) e = cudaMemcpyAsync(r.weights, f + data_off, size - data_off, cudaMemcpyHostToDevice, r.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(r.stream);
    if (e != cudaSuccess) {
      set_error("%s: %suploading %s: %s", who, at, path, cudaGetErrorString(e));
      return fail(-2);
    }
    bind_weights(r, specs, lay, outdim, precision == SOME_PRECISION_FP32, [&](const std::string& name) -> const void* {
      return static_cast<uint8_t*>(r.weights) + (dir.at(name).off - data_off);
    });
    r.model.b_cut = r.model32.b_cut = rd<float>(f + dir.at("b_cut").off);   // a host scalar of the model
    r.pool.reset(new WorkerPool(lanes));
  }
  s->stream = s->reps[0]->stream;
  s->pool = s->reps[0]->pool.get();
  s->load.assign(n, {0, 0});
  s->lanes.reset(new WorkerPool(n));      // one replica: no thread, its lane runs on the calling thread
  if (n > 1) {
    DeviceScope scope(s->device);
    e = cudaEventCreateWithFlags(&s->fed, cudaEventDisableTiming);
    if (e != cudaSuccess) {
      set_error("%s: cudaEventCreate: %s", who, cudaGetErrorString(e));
      return fail(-2);
    }
  }
  const Entry& kt = dir.at("kaiser_best");
  s->kaiser.resize(kKaiserTaps);
  memcpy(s->kaiser.data(), f + kt.off, kt.bytes);
  s->info.sample_rate = sr;
  s->info.hop = hop;
  s->info.outdim = outdim;
  s->info.quantized = quantized;
  s->info.bias_corrected = bias_corrected;
  s->precision = precision;
  s->info.timestep = static_cast<double>(hop) / static_cast<double>(sr);    // base_infer.py:20
  s->vmin = rd<float>(f + 60), s->vmax = rd<float>(f + 64), s->deviation = rd<float>(f + 68), s->threshold = rd<float>(f + 72);
  *out = s;
  return 0;
}
}  // namespace

extern "C" int some_session_open(const char* path, int device, some_session** out) {
  SOME_REQUIRE(path != nullptr && out != nullptr, "some_session_open: null pointer");
  *out = nullptr;
  return open_session("some_session_open", path, &device, 1, false, out);
}

extern "C" int some_session_open_devices(const char* path, const int* devices, int n, some_session** out) {
  const char* who = "some_session_open_devices";
  SOME_REQUIRE(path != nullptr && out != nullptr, "%s: null pointer", who);
  *out = nullptr;
  SOME_REQUIRE(devices != nullptr, "%s: the device list is NULL", who);
  SOME_REQUIRE(n >= 1 && n <= kMaxReplicas, "%s: %d devices (1 to %d)", who, n, kMaxReplicas);
  for (int i = 0; i < n; ++i) SOME_REQUIRE(devices[i] >= 0, "%s: devices[%d] is %d", who, i, devices[i]);
  return open_session(who, path, devices, n, true, out);
}

extern "C" int some_session_get_devices(const some_session* s, int* devices, int capacity, int* n) {
  SOME_REQUIRE(s != nullptr && n != nullptr && capacity >= 0 && (capacity == 0 || devices != nullptr),
               "some_session_get_devices: bad arguments");
  *n = static_cast<int>(s->reps.size());
  for (int i = 0; i < std::min(capacity, *n); ++i) devices[i] = s->reps[i]->device;
  return 0;
}

extern "C" int some_session_get_load(const some_session* s, int64_t* chunks, int64_t* frames, int capacity, int* n) {
  SOME_REQUIRE(s != nullptr && n != nullptr && capacity >= 0 && (capacity == 0 || (chunks != nullptr && frames != nullptr)),
               "some_session_get_load: bad arguments");
  std::lock_guard<std::mutex> lock(s->mu);
  *n = static_cast<int>(s->load.size());
  for (int i = 0; i < std::min(capacity, *n); ++i) chunks[i] = s->load[i].first, frames[i] = s->load[i].second;
  return 0;
}

extern "C" int some_session_get_stats(const some_session* s, some_session_stats* stats) {
  SOME_REQUIRE(s != nullptr && stats != nullptr, "some_session_get_stats: null pointer");
  std::lock_guard<std::mutex> lock(s->mu);
  *stats = s->stats;
  stats->queued = static_cast<int64_t>(s->queue.size());
  return 0;
}

extern "C" int some_shard_clips(const int64_t* lens, int n, int replicas, int32_t* owner) {
  SOME_REQUIRE(n >= 0 && replicas >= 1 && (n == 0 || (lens != nullptr && owner != nullptr)), "some_shard_clips: bad arguments");
  // clip_cost of some_b200/dist.py: T frames cost T * (dense + attention * T); 16384 * T is exact, so no rounding depends on
  // how the compiler contracts the expression
  std::vector<double> cost(n);
  for (int i = 0; i < n; ++i) {
    SOME_REQUIRE(lens[i] >= 0, "some_shard_clips: clip %d has a negative length", i);
    const double t = static_cast<double>(1 + lens[i] / SOME_HOP);
    cost[i] = t * (103.31e6 + 16384.0 * t);
  }
  std::vector<int> order(n);
  for (int i = 0; i < n; ++i) order[i] = i;
  std::sort(order.begin(), order.end(), [&](int a, int b) { return cost[a] != cost[b] ? cost[a] > cost[b] : a < b; });
  std::vector<double> load(replicas, 0.0);
  for (int i : order) {                   // longest first, to the least loaded replica (ties: the lowest)
    int best = 0;
    for (int r = 1; r < replicas; ++r)
      if (load[r] < load[best]) best = r;
    owner[i] = best;
    load[best] += cost[i];
  }
  return 0;
}

extern "C" int some_session_close(some_session* s) {
  if (s) destroy(s);
  return 0;
}

extern "C" int some_session_get_info(const some_session* s, some_session_info* info) {
  SOME_REQUIRE(s != nullptr && info != nullptr, "some_session_get_info: null pointer");
  *info = s->info;
  return 0;
}

extern "C" int some_session_get_precision(const some_session* s, int* precision) {
  SOME_REQUIRE(s != nullptr && precision != nullptr, "some_session_get_precision: null pointer");
  *precision = s->precision;
  return 0;
}

namespace {
// resampy's refusal: a recording of n samples at `rate` whose output at the model's rate sr would be empty.
bool too_short_to_resample(int64_t n, int rate, int sr) { return rate != sr && n * sr / rate < 1; }

// What the slicer sees of a recording of n samples at sample_rate: its length at the model's rate (audio.resampled_length:
// librosa.load's output length; resampy refuses a recording whose own output would be empty) and, unless the recording is
// one chunk anyway, the number of RMS frames to cut it by.
struct SliceShape {
  int64_t n_out = 0;
  int frames = 0;       // 0: one chunk [0, n_out)
};
int slice_shape(int64_t n, int sample_rate, int sr, const some_slicer_frames& sl, const char* who, SliceShape* sh) {
  SOME_REQUIRE(!too_short_to_resample(n, sample_rate, sr), "%s: Input signal length=%lld is too small to resample from %d->%d",
               who, static_cast<long long>(n), sample_rate, sr);
  sh->n_out = n;
  if (sample_rate != sr) sh->n_out = static_cast<int64_t>(ceil(static_cast<double>(n) * (static_cast<double>(sr) / sample_rate)));
  const int64_t frames = frames_whole(sl, sh->n_out);
  SOME_REQUIRE(frames < (int64_t(1) << 31), "%s: recording too long", who);
  sh->frames = static_cast<int>(frames);
  return 0;
}
// The chunk ranges of a recording from its shape and, when it is cut, its sh.frames RMS values.
int slice_ranges(const SliceShape& sh, const float* rms, const some_slicer_frames& sl, std::vector<int64_t>& ranges) {
  if (sh.frames == 0) {
    ranges = {0, sh.n_out};
    return 0;
  }
  ranges.resize(2 * (static_cast<size_t>(sh.frames) + 2));
  int count = 0;
  if (some_slicer_ranges(rms, sh.frames, sh.n_out, &sl, ranges.data(), sh.frames + 2, &count)) return -1;
  ranges.resize(2 * static_cast<size_t>(count));
  return 0;
}

// A recording of a sliced or an encoded call: host floats (`host`, the sliced call) or a file's bytes (the encoded call).
struct RecItem {
  const float* host = nullptr;
  const uint8_t* bytes = nullptr;
  const some_device_audio* dev = nullptr;   // the device call: its item, the item's layout and the event its producer recorded
  int layout = 0;
  cudaEvent_t ready = nullptr;
  some_audio_meta m{};        // of the file; the sliced call sets only its rate
  int64_t n = 0;              // samples at its rate (FLAC without a stated length: known after the chain)
  SliceShape sh;
  some_notes* out = nullptr;
  int64_t up = 0;             // the audio bytes' offset in the upload
};
struct StepItem;
struct ByteItem;
struct PeekItem;

// One public call, queued for a step (see submit): what it asks for, what it touches and, once its step has run, its result.
struct Request {
  enum Kind { CLIPS, RECORDINGS, STREAMS, BYTES, PEEKS } kind;
  int pdl = 0;                            // the caller's some_set_pdl setting
  int64_t samples = 0;                    // the model-rate samples it adds to a step (streams: see some_session_stats)
  bool sized = true;                      // false: its size is not known before the GPU work (it takes no joiners)
  std::vector<const void*> touches;       // its streams and its some_notes
  // the work, by kind: CLIPS
  const float* const* clips = nullptr;
  const int64_t* lens = nullptr;
  int B = 0;
  some_notes* out = nullptr;
  // RECORDINGS (the sliced call: one host item) with the slicer's frames, STREAMS, BYTES, PEEKS
  std::vector<RecItem>* recs = nullptr;
  some_slicer_frames sl{};
  std::vector<StepItem>* items = nullptr;
  std::vector<ByteItem>* bytes = nullptr;
  std::vector<PeekItem>* peeks = nullptr;
  // the result
  int rc = 0;
  std::string err;
  bool done = false;
  void fail(int code, const std::string& message) {
    if (rc == 0) rc = code, err = message;
  }
};
int submit(some_session* s, Request& rq);

// The resampling table for sample_rate -> the model's rate: uploaded on the session's stream (in front of the resampling
// launches that read it) the first time its ratio is used, and kept.  Upsampling reads the table as it is; resampy scales it
// by the ratio when downsampling (audio._device_table), so each downsampling ratio has its own copy.
const double* table_for(some_session* s, int sample_rate) {
  const double ratio = static_cast<double>(s->info.sample_rate) / sample_rate;
  some_session::Table& t = s->tables[ratio < 1 ? ratio : 1.0];
  if (t.d.cap == 0) {
    t.h = s->kaiser;
    if (ratio < 1)
      for (double& v : t.h) v = ratio * v;
    if (t.d.ensure(8ull * kKaiserTaps, "the resampling table")) return nullptr;
    const cudaError_t e = cudaMemcpyAsync(t.d.p, t.h.data(), 8ull * kKaiserTaps, cudaMemcpyHostToDevice, s->stream);
    if (e != cudaSuccess) {
      set_error("session: table upload: %s", cudaGetErrorString(e));
      t.d.release();
      return nullptr;
    }
  }
  return static_cast<const double*>(t.d.p);
}

// The host-to-device copy of a step's samples and descriptors: regions of the session's pinned step_h, each 16-byte aligned,
// filled once reserve() has made room for all of them, and sent to the same offsets of step_d in one copy.
struct Upload {
  some_session* s;
  size_t bytes = 0;
  size_t add(size_t n) {
    const size_t off = bytes;
    bytes += align16(n);
    return off;
  }
  int reserve(const char* what) { return s->step_h.ensure(bytes, what) || s->step_d.ensure(bytes, what) ? -1 : 0; }
  char* h(size_t off) const { return static_cast<char*>(s->step_h.p) + off; }
  char* d(size_t off) const { return static_cast<char*>(s->step_d.p) + off; }
  int send(const char* what) const {
    if (bytes) SOME_CUDA(cudaMemcpyAsync(s->step_d.p, s->step_h.p, bytes, cudaMemcpyHostToDevice, s->stream), what);
    return 0;
  }
};

// The resampling and RMS windows of a step, launched together on the session's stream:
//   rms     adds an RMS window and returns where its first frame lies in the session's RMS buffers (after the frames of the
//           windows added before it);
//   place   after every other region of the step's upload is added: a descriptor region for each kind that has windows (so
//           a step without any uploads nothing for them), the upload reserved, the RMS buffers sized and the descriptors packed;
//   launch  after the upload is sent and the samples are written: one resampling launch, one RMS launch, the RMS download.
struct StepWindows {
  std::vector<some_resample_window> rs;
  std::vector<some_rms_window> rm;
  int64_t frames = 0;
  size_t rs_off = 0, rm_off = 0;

  int64_t rms(const some_rms_window& w) {
    const int64_t at = frames;
    rm.push_back(w);
    frames += w.f_end - w.f_begin;
    return at;
  }

  int place(some_session* s, Upload& up, const char* what) {
    const int kr = static_cast<int>(rs.size()), km = static_cast<int>(rm.size());
    if (kr) rs_off = up.add(static_cast<size_t>(some_resample_windows_bytes(kr)));
    if (km) rm_off = up.add(static_cast<size_t>(some_slicer_rms_windows_bytes(km)));
    if (up.reserve(what) || s->rms_d.ensure(4ull * frames + 16, "the RMS frames") ||
        s->rms_h.ensure(4ull * frames + 16, "the RMS frames"))
      return -1;
    float* at = static_cast<float*>(s->rms_d.p);
    for (some_rms_window& w : rm) w.rms = at, at += w.f_end - w.f_begin;
    if ((kr && some_resample_windows_pack(rs.data(), kr, up.h(rs_off))) ||
        (km && some_slicer_rms_windows_pack(rm.data(), km, up.h(rm_off))))
      return -1;
    return 0;
  }

  int launch(some_session* s, const Upload& up) const {
    if ((!rs.empty() && some_resample_kaiser_windows(up.h(rs_off), up.d(rs_off), s->stream)) ||
        (!rm.empty() && some_slicer_rms_windows(up.h(rm_off), up.d(rm_off), s->stream)))
      return -1;
    if (frames)
      SOME_CUDA(cudaMemcpyAsync(s->rms_h.p, s->rms_d.p, 4ull * frames, cudaMemcpyDeviceToHost, s->stream), "RMS download");
    return 0;
  }
};

// The device audio of a step (some_session_transcribe_device, some_stream_push_device*), down-mixed by one some_downmix launch
// into the session's buffers:
//   add     the descriptor region of k items in the step's upload;
//   push    an item, with where its frames mono samples go (on the session's device) and the event its producer recorded;
//   fill    after every push: room for the packed copies of the items on other devices, and the descriptors;
//   launch  after the upload is sent: the session's stream waits on every item's event, copies the items on other devices
//           (cudaMemcpyPeerAsync: channel c of a planar item to c * frames) and launches the down-mix.
struct Downmix {
  std::vector<some_downmix_item> items;
  std::vector<const some_device_audio*> src;
  std::vector<cudaEvent_t> ready;
  size_t off = 0;
  int k = 0;

  void add(Upload& up, int count) {
    k = count;
    if (k) off = up.add(static_cast<size_t>(some_downmix_bytes(k)));
  }
  void push(const some_device_audio& a, int layout, cudaEvent_t ev, float* out) {
    items.push_back(some_downmix_item{a.data, a.frames, a.channels, layout, a.channel_stride, out});
    src.push_back(&a), ready.push_back(ev);
  }
  // A copied item's channels lie `rows` floats apart (rows 0: the item is copied as one block).
  static int64_t rows(const some_downmix_item& it) {
    if (it.channels == 1) return 0;
    return it.layout == SOME_DOWNMIX_PLANAR ? it.frames : it.layout == SOME_DOWNMIX_INTERLEAVED && it.frames == 1 ? 1 : 0;
  }
  bool remote(const some_session* s, size_t j) const { return src[j]->device != s->device && items[j].frames > 0; }
  int fill(some_session* s, const Upload& up) {
    SOME_REQUIRE(static_cast<int>(items.size()) == k, "session: %zu device items, %d placed", items.size(), k);
    if (k == 0) return 0;
    int64_t total = 0;
    for (size_t j = 0; j < items.size(); ++j)
      if (remote(s, j)) total += align4(items[j].frames * items[j].channels);
    if (total && s->peer_d.ensure(4ull * total + 16, "the copies of device audio")) return -1;
    float* at = static_cast<float*>(s->peer_d.p);
    for (size_t j = 0; j < items.size(); ++j)
      if (remote(s, j)) {
        some_downmix_item& it = items[j];
        it.data = at;
        if (rows(it)) it.channel_stride = rows(it);
        at += align4(it.frames * it.channels);
      }
    return some_downmix_pack(items.data(), k, up.h(off));
  }
  int launch(some_session* s, const Upload& up) const {
    if (k == 0) return 0;
    for (cudaEvent_t e : ready)
      if (e) SOME_CUDA(cudaStreamWaitEvent(s->stream, e, 0), "waiting for the device audio's stream");
    for (size_t j = 0; j < items.size(); ++j) {
      if (!remote(s, j)) continue;
      const some_device_audio& a = *src[j];
      const some_downmix_item& it = items[j];
      float* dst = const_cast<float*>(it.data);
      const int64_t r = rows(it);
      if (r) {
        for (int c = 0; c < it.channels; ++c)
          SOME_CUDA(cudaMemcpyPeerAsync(dst + c * r, s->device, a.data + c * a.channel_stride, a.device, 4ull * r, s->stream),
                    "device audio copy");
      } else {
        SOME_CUDA(cudaMemcpyPeerAsync(dst, s->device, a.data, a.device, 4ull * it.frames * it.channels, s->stream),
                  "device audio copy");
      }
    }
    return some_downmix(up.h(off), up.d(off), s->stream);
  }
};

// Recordings in the session's recording buffer, each at its own rate and with its own slicer frames, made into chunks and
// notes together (the sliced and the encoded calls of a step; the step writes the recordings there and may add its own regions
// to the upload and its own launches and downloads in front of the synchronise):
//   place   where each recording and its model-rate samples go; one resampling window per recording at another rate and one
//           RMS window per recording that is cut, placed in the upload after the caller's own regions (the caller fills its
//           regions after this, and launches the windows once the upload is sent and the recordings are written);
//   finish  after the caller's synchronise: each recording's cuts, one batch over all chunks, each recording's notes (a
//           recording whose `out` has been set to NULL since place, its call refused, is left out).
struct Recordings {
  struct Item {
    int rate;
    int64_t n;                // samples at `rate`
    SliceShape sh;
    const some_slicer_frames* sl;
    some_notes* out;
    int64_t x = 0, y = 0;     // its samples at `rate` and at the model's rate in the buffer (the same at the model's rate)
    int64_t rms0 = 0;         // its first RMS frame
    int c0 = 0, c1 = 0;       // its chunks in the batch
  };
  std::vector<Item> items;
  float* base = nullptr;      // the recording buffer
  StepWindows win;

  int place(some_session* s, Upload& up) {
    const int sr = s->info.sample_rate;
    int64_t total = 0;
    for (Item& it : items) {
      it.x = it.y = total;
      total += align4(it.n);
      if (it.rate != sr) it.y = total, total += align4(it.sh.n_out);
    }
    if (s->rec_d.ensure(4ull * total + 16, "the recordings")) return -1;
    base = static_cast<float*>(s->rec_d.p);
    for (Item& it : items) {
      if (it.rate != sr) {
        const double* table = table_for(s, it.rate);
        if (!table) return -1;
        win.rs.push_back({base + it.x, 0, it.n, 1, base + it.y, 0, 0, it.sh.n_out, it.rate, sr, table, kKaiserTaps});
      }
      if (it.sh.frames)
        it.rms0 = win.rms({base + it.y, 0, it.sh.n_out, it.sh.n_out, it.sl->win_size, it.sl->hop_size, nullptr, 0, it.sh.frames});
    }
    return win.place(s, up, "the step's upload");
  }

  int finish(some_session* s) {
    std::vector<int64_t> starts, lens, begin, ranges;
    for (Item& it : items) {
      if (!it.out) continue;
      if (slice_ranges(it.sh, static_cast<const float*>(s->rms_h.p) + it.rms0, *it.sl, ranges)) return -1;
      it.c0 = static_cast<int>(starts.size());
      for (size_t r = 0; r + 1 < ranges.size(); r += 2) {
        begin.push_back(ranges[r]);
        starts.push_back(it.y + ranges[r]);
        lens.push_back(std::max<int64_t>(0, ranges[r + 1] - ranges[r]));
      }
      it.c1 = static_cast<int>(starts.size());
    }
    const int B = static_cast<int>(starts.size());
    if (B && run_chunks(s, nullptr, base, starts.data(), lens.data(), B)) return -1;
    for (const Item& it : items)
      if (it.out) take_chunks(s, it.c0, it.c1, begin.data(), lens.data(), it.out);
    return 0;
  }
};

}  // namespace

extern "C" int some_session_transcribe(some_session* s, const float* const* clips, const int64_t* lens, int B, some_notes* out) {
  SOME_REQUIRE(s != nullptr && out != nullptr && B >= 0 && (B == 0 || (clips != nullptr && lens != nullptr)),
               "some_session_transcribe: bad arguments");
  for (int i = 0; i < B; ++i) SOME_REQUIRE(lens[i] >= 0 && (lens[i] == 0 || clips[i] != nullptr), "some_session_transcribe: clip %d", i);
  if (B == 0) {
    clear(out);
    return 0;
  }
  Request rq{Request::CLIPS};
  rq.clips = clips, rq.lens = lens, rq.B = B, rq.out = out;
  for (int i = 0; i < B; ++i) rq.samples += lens[i];
  rq.touches = {out};
  return submit(s, rq);
}

extern "C" int some_session_transcribe_sliced(some_session* s, const float* samples, long long n, int sample_rate,
                                              const some_slicer_params* params, some_notes* out) {
  SOME_REQUIRE(s != nullptr && out != nullptr && n >= 0 && (n == 0 || samples != nullptr) && sample_rate > 0,
               "some_session_transcribe_sliced: bad arguments");
  const int sr = s->info.sample_rate;
  some_slicer_frames sl;
  if (some_slicer_derive(sr, params, &sl)) return -1;
  std::vector<RecItem> recs(1);
  RecItem& it = recs[0];
  if (slice_shape(n, sample_rate, sr, sl, "some_session_transcribe_sliced", &it.sh)) return -1;
  it.host = samples, it.m.rate = sample_rate, it.n = n, it.out = out;
  Request rq{Request::RECORDINGS};
  rq.recs = &recs, rq.sl = sl, rq.samples = it.sh.n_out, rq.touches = {out};
  return submit(s, rq);
}

// ---------------------------------------------------------------------------------------------------- streams
namespace {
// Samples [first, first + len) of an unbounded sequence, at buf + off in a device buffer.
struct SampleWindow {
  DevBuf buf;
  int64_t first = 0, len = 0, off = 0;
  float* at(int64_t i) const { return static_cast<float*>(buf.p) + off + (i - first); }
  // Drops the samples before `keep` and makes room for n more after the window.  When the buffer's end is reached, the kept
  // samples move to its front in one device-to-device copy on `stream`, or into a larger buffer when they would overlap
  // themselves there or leave no room.
  int reserve(cudaStream_t stream, int64_t keep, int64_t n, const char* what) {
    keep = std::min(std::max(keep, first), first + len);
    off += keep - first, len -= keep - first, first = keep;
    const int64_t cap = static_cast<int64_t>(buf.cap / 4);
    if (buf.p && off + len + n <= cap) return 0;
    if (buf.p && len + n <= cap && len <= off) {
      if (len) SOME_CUDA(cudaMemcpyAsync(buf.p, at(first), 4ull * len, cudaMemcpyDeviceToDevice, stream), "stream compaction");
      off = 0;
      return 0;
    }
    DevBuf bigger;
    if (bigger.ensure(4ull * std::max<int64_t>(2 * (len + n), 1 << 16), what)) return -1;
    if (len) SOME_CUDA(cudaMemcpyAsync(bigger.p, at(first), 4ull * len, cudaMemcpyDeviceToDevice, stream), "stream compaction");
    SOME_CUDA(cudaStreamSynchronize(stream), "synchronise");
    buf = std::move(bigger);
    off = 0;
    return 0;
  }
};
// The upload scatter of a stream step: entry j copies n samples of the step's device upload into a stream's window.
struct ScatterParams {
  const float* src;
  float* dst;
  long long n;
};
constexpr int kScatterThreads = 256, kScatterTile = 8 * kScatterThreads;

__global__ void __launch_bounds__(kScatterThreads) scatter_kernel(const ScatterParams* __restrict__ ps,
                                                                  const long long* __restrict__ tile0, int K) {
  const long long tile = blockIdx.x;
  const int w = window_of(tile0, K, tile);
  const ScatterParams& p = ps[w];
  const long long e = min(p.n, (tile - tile0[w] + 1) * kScatterTile);
  for (long long i = (tile - tile0[w]) * kScatterTile + threadIdx.x; i < e; i += kScatterThreads) p.dst[i] = __ldg(p.src + i);
}
}  // namespace

struct some_stream {
  some_session* s = nullptr;
  int rate = 0;                           // of the pushed samples
  bool resample = false;
  some_slicer_stream* slicer = nullptr;   // the slicer's decisions (some_slicer_stream_*)
  some_slicer_frames f{};                 // its frame counts
  SampleWindow native, wave;              // the input at its own rate (when resampling) and at the model's rate
  DevBuf head_d;                          // model-rate samples [0, head_len) kept apart during a long leading silence
  int64_t head_len = 0;
  int64_t received = 0, fixed = 0, frames = 0;   // frames: RMS frames computed so far
  bool finished = false;
  // an encoded stream (some_stream_open_encoded; rate 0 until its header is complete): the container walk, the audio bytes
  // not decoded yet (file offsets [pend_pos, pend_pos + size): an incomplete FLAC frame or WAV or AIFF sample frame) and the chain
  std::unique_ptr<AudioWalk> walk;
  bool failed = false;                    // refused on its content
  std::vector<uint8_t> pending;
  long long pend_pos = 0;
  FlacWalk fw;
};

namespace {
void destroy(some_stream* st) {
  some_slicer_stream_destroy(st->slicer);
  DeviceScope scope(st->s->device);
  delete st;                              // its buffers free themselves, on the session's device
}

// One stream's part of a step: n new samples, whether the recording ends there, and where its chunks go.
struct StepItem {
  some_stream* st;
  const float* samples;
  int64_t n;
  bool final;
  some_notes* out;
  const some_device_audio* dev = nullptr;   // a device push: its item (n = its frames), layout and producer's event
  int layout = 0;
  cudaEvent_t ready = nullptr;
  int64_t up = 0;               // where its samples lie in the upload (floats)
  int64_t rms0 = 0, nf = 0;     // its new RMS frames in the session's RMS buffer
  int c0 = 0, c1 = 0;           // its chunks in the step's batch
  bool dropped = false;         // its samples failed to decode: no slicer decisions, no chunks
  std::string why;              // and the decoder's message
};

// Whether a container's samples are PCM that some_pcm_decode reads (WAV, AIFF) rather than FLAC frames: the one place the
// encoded calls tell the two paths apart.
bool pcm_container(const some_audio_meta& m) { return m.container != SOME_AUDIO_FLAC; }

// Accepts audio at `rate` for a session at rate `sr`, or refuses a rate pair the resampler does not support (with
// some_resample_window_plan's message).
int check_rates(int rate, int sr) {
  long long t_end, x_first;
  return rate != sr && some_resample_window_plan(0, 0, 0, rate, sr, kKaiserTaps, &t_end, &x_first) ? -1 : 0;
}

// Accepts a container's format for a session at rate `sr`, or refuses it (the message has no prefix): a PCM file's mono
// down-mix takes at most 128 channels, and the resampler must support the rate pair.
int check_format(const some_audio_meta& m, int sr) {
  SOME_REQUIRE(!pcm_container(m) || m.channels <= 128, "a mono down-mix of %d channels (at most 128)", m.channels);
  return check_rates(m.rate, sr);
}
// One window of a call's audio bytes (a file's data chunk, a stream's pending bytes), with its container's metadata.
struct ByteWindow {
  const some_audio_meta* m;
  const uint8_t* src;
  int64_t bytes;
  int64_t* at;                                   // out: its offset in the bytes upload
};

// The encoded-input stage of the encoded calls (some_session_transcribe_encoded and the encoded stream step): the audio bytes
// go up, FLAC frames are found on the device and chained on the host by the caller, and the samples are decoded, mono, into
// the caller's buffer.
//   upload  the windows, FLAC first (the scan covers only them), each 16-byte aligned, then one some_flac_stream per FLAC
//           window: copied into pinned memory in pieces of up to 1 MB and sent in one copy;
//   scan    with FLAC windows: one some_flac_scan and the candidates down, again with room for all if the estimate was short;
//   add     the regions of the PCM descriptors, the chained FLAC frames (their scratch and output offsets) and the status
//           word in the caller's descriptor upload;
//   fill    after the caller has placed each item's samples: the descriptors, with those places;
//   launch  after the descriptor upload is sent: one some_pcm_decode, one FLAC decode, the status download;
//   check   after the synchronise: every item whose frame failed to decode, each with its message.
struct Decode {
  const uint8_t* bytes_d = nullptr;              // the bytes upload
  int64_t flac_bytes = 0;                        // its FLAC windows: [0, flac_bytes), described by streams_d[0 .. nf)
  int nf = 0;
  const some_flac_stream* streams_d = nullptr;
  const some_flac_frame* frames_h = nullptr;     // the candidates, on the host and on the device
  const some_flac_frame* frames_d = nullptr;
  int n_cand = 0;
  std::vector<some_pcm_item> pcm;                // out: set by fill()
  std::vector<int> pcm_of, flac_of;              // the caller's item of each PCM entry and of each FLAC window
  std::vector<int64_t> first{0};                 // FLAC window r's frames: chain[first[r] .. first[r + 1])
  std::vector<int32_t> chain;
  std::vector<int> channels;
  std::vector<long long> base;                   // FLAC window r: file offset x lies at x + base[r] in the bytes upload
  float* out = nullptr;                          // fill(): the FLAC windows' output base
  size_t pcm_off = 0, chain_off = 0, soff_off = 0, ooff_off = 0, status_off = 0;

  int upload(some_session* s, const std::vector<ByteWindow>& ws, const char* what) {
    int64_t at = 0;
    auto place = [&](bool flac) {
      for (const ByteWindow& w : ws)
        if (!pcm_container(*w.m) == flac) *w.at = at, at += align16(w.bytes), nf += flac;
    };
    place(true);
    flac_bytes = at;
    place(false);
    const int64_t up_bytes = at + static_cast<int64_t>(sizeof(some_flac_stream)) * nf;
    if (s->enc_h.ensure(up_bytes + 16, what) || s->enc_d.ensure(up_bytes + 16, what)) return -1;
    uint8_t* up_h = static_cast<uint8_t*>(s->enc_h.p);
    std::vector<HostSpan> spans;
    some_flac_stream* st_h = reinterpret_cast<some_flac_stream*>(up_h + at);
    for (const ByteWindow& w : ws) {
      spans.push_back({up_h + *w.at, w.src, static_cast<size_t>(w.bytes)});
      if (!pcm_container(*w.m))
        *st_h++ = some_flac_stream{*w.at, *w.at + w.bytes, w.m->channels, w.m->bits, w.m->max_blocksize, 0};
    }
    copy_to_pinned(*s->pool, spans, size_t(1) << 20);
    bytes_d = static_cast<const uint8_t*>(s->enc_d.p);
    streams_d = reinterpret_cast<const some_flac_stream*>(bytes_d + at);
    if (up_bytes) SOME_CUDA(cudaMemcpyAsync(s->enc_d.p, up_h, static_cast<size_t>(up_bytes), cudaMemcpyHostToDevice, s->stream),
                            "encoded upload");
    return 0;
  }
  // `cap`: the caller's estimate of the candidates.  with_count: all `cap` come down with the count, in one synchronise;
  // otherwise the count comes down first, then exactly that many.
  int scan(some_session* s, int64_t cap, bool with_count) {
    const uint64_t ws_bytes = some_flac_scan_workspace_bytes(flac_bytes);
    if (s->flac_ws_d.ensure(ws_bytes + 16, "the FLAC scan workspace")) return -1;
    int* count_d = reinterpret_cast<int*>(static_cast<char*>(s->flac_ws_d.p) + ws_bytes);
    char* fh;                                    // the count, then the candidates at fh + 16
    for (;;) {
      if (s->flac_frames_d.ensure(sizeof(some_flac_frame) * cap, "the FLAC frames") ||
          s->flac_frames_h.ensure(sizeof(some_flac_frame) * cap + 16, "the FLAC frames"))
        return -1;
      fh = static_cast<char*>(s->flac_frames_h.p);
      if (some_flac_scan(bytes_d, flac_bytes, streams_d, nf, static_cast<some_flac_frame*>(s->flac_frames_d.p),
                         static_cast<int>(cap), count_d, s->flac_ws_d.p, s->stream))
        return -1;
      SOME_CUDA(cudaMemcpyAsync(fh, count_d, sizeof(int), cudaMemcpyDeviceToHost, s->stream), "count download");
      if (with_count)
        SOME_CUDA(cudaMemcpyAsync(fh + 16, s->flac_frames_d.p, sizeof(some_flac_frame) * cap, cudaMemcpyDeviceToHost,
                                  s->stream), "candidate download");
      SOME_CUDA(cudaStreamSynchronize(s->stream), "synchronise");
      n_cand = *reinterpret_cast<const int*>(fh);
      if (n_cand <= cap) break;
      cap = n_cand;
    }
    if (!with_count) {
      SOME_CUDA(cudaMemcpyAsync(fh + 16, s->flac_frames_d.p, sizeof(some_flac_frame) * n_cand, cudaMemcpyDeviceToHost,
                                s->stream), "candidate download");
      SOME_CUDA(cudaStreamSynchronize(s->stream), "synchronise");
    }
    frames_h = reinterpret_cast<const some_flac_frame*>(fh + 16);
    frames_d = static_cast<const some_flac_frame*>(s->flac_frames_d.p);
    return 0;
  }
  void add(Upload& up) {
    const size_t n = chain.size();
    pcm_off = up.add(static_cast<size_t>(some_pcm_decode_bytes(static_cast<int>(pcm.size()))));
    chain_off = up.add(4 * n), soff_off = up.add(8 * n), ooff_off = up.add(8 * n), status_off = up.add(2 * sizeof(int));
  }
  // item i's samples go to dst + at(i)
  template <class At>
  int fill(some_session* s, const Upload& up, float* dst, At at) {
    out = dst;
    for (size_t j = 0; j < pcm.size(); ++j) pcm[j].out = dst + at(pcm_of[j]);
    int64_t* soff = reinterpret_cast<int64_t*>(up.h(soff_off));
    int64_t* ooff = reinterpret_cast<int64_t*>(up.h(ooff_off));
    int64_t scratch = 0;
    for (size_t r = 0; r < flac_of.size(); ++r) {
      int64_t o = at(flac_of[r]);
      for (int64_t j = first[r]; j < first[r + 1]; ++j) {
        const int bs = frames_h[chain[j]].blocksize;
        soff[j] = scratch, ooff[j] = o;
        scratch += static_cast<int64_t>(bs) * channels[r], o += bs;
      }
    }
    if (s->flac_scratch_d.ensure(4ull * scratch + 16, "the FLAC scratch") ||
        some_pcm_decode_pack(pcm.data(), static_cast<int>(pcm.size()), up.h(pcm_off)))
      return -1;
    if (!chain.empty()) memcpy(up.h(chain_off), chain.data(), 4 * chain.size());
    int* status = reinterpret_cast<int*>(up.h(status_off));
    status[0] = 0, status[1] = INT_MAX;          // the first chained frame that fails to decode, if one does
    return 0;
  }
  int launch(some_session* s, const Upload& up) const {
    if (some_pcm_decode(up.h(pcm_off), up.d(pcm_off), s->stream)) return -1;
    if (chain.empty()) return 0;
    int* status_d = reinterpret_cast<int*>(up.d(status_off));
    if (flac_decode_chain(bytes_d, streams_d, frames_d, reinterpret_cast<const int32_t*>(up.d(chain_off)),
                          reinterpret_cast<const int64_t*>(up.d(soff_off)), reinterpret_cast<const int64_t*>(up.d(ooff_off)),
                          static_cast<int>(chain.size()), static_cast<int32_t*>(s->flac_scratch_d.p), out, 1, status_d,
                          status_d + 1, s->stream))
      return -1;
    SOME_CUDA(cudaMemcpyAsync(up.h(status_off), status_d, 2 * sizeof(int), cudaMemcpyDeviceToHost, s->stream), "status download");
    return 0;
  }
  // The caller's items whose frame failed to decode, each with the message of its first such frame (the frame's byte offset
  // in its file), in window order.  The status word names the first failing frame of a launch, so after each failure the
  // frames of the later windows are decoded again, with a fresh status word, until none fails (into the same places, with
  // the same values: only the status is new).
  int check(some_session* s, const Upload& up, std::vector<std::pair<int, std::string>>& failed) const {
    int* status = reinterpret_cast<int*>(up.h(status_off));
    int* status_d = reinterpret_cast<int*>(up.d(status_off));
    int64_t k = 0;                               // the launch checked covers chain[k ..)
    while (!chain.empty() && status[0] != 0) {
      const int64_t j = k + status[1];
      size_t r = 0;
      while (r + 1 < flac_of.size() && first[r + 1] <= j) ++r;
      char msg[160];
      snprintf(msg, sizeof(msg), "FLAC frame at byte offset %lld failed to decode (status %d)",
               static_cast<long long>(frames_h[chain[j]].pos - base[r]), status[0]);
      failed.push_back({flac_of[r], msg});
      k = first[r + 1];
      if (k >= static_cast<int64_t>(chain.size())) break;
      status[0] = 0, status[1] = INT_MAX;
      SOME_CUDA(cudaMemcpyAsync(status_d, status, 2 * sizeof(int), cudaMemcpyHostToDevice, s->stream), "status upload");
      if (flac_decode_chain(bytes_d, streams_d, frames_d, reinterpret_cast<const int32_t*>(up.d(chain_off)) + k,
                            reinterpret_cast<const int64_t*>(up.d(soff_off)) + k, reinterpret_cast<const int64_t*>(up.d(ooff_off)) + k,
                            static_cast<int>(chain.size() - k), static_cast<int32_t*>(s->flac_scratch_d.p), out, 1, status_d,
                            status_d + 1, s->stream))
        return -1;
      SOME_CUDA(cudaMemcpyAsync(status, status_d, 2 * sizeof(int), cudaMemcpyDeviceToHost, s->stream), "status download");
      SOME_CUDA(cudaStreamSynchronize(s->stream), "synchronise");
    }
    return 0;
  }
};

// Device-resident ranges of the session's streams (src[c]: lens[c] samples on replica 0's device), copied next to each other
// into replica 0's audio buffer on the session's stream and transcribed as one batch.
int run_resident(some_session* s, const std::vector<const float*>& src, const std::vector<int64_t>& lens) {
  const int B = static_cast<int>(lens.size());
  if (B == 0) return 0;
  std::vector<int64_t> starts(B);
  int64_t total = 0;
  for (int c = 0; c < B; ++c) starts[c] = total, total += align4(lens[c]);
  DevBuf& chunks_d = s->reps[0]->wave_d;
  if (chunks_d.ensure(4ull * total + 16, "the audio")) return -1;
  float* wave = static_cast<float*>(chunks_d.p);
  for (int c = 0; c < B; ++c)
    if (lens[c])
      SOME_CUDA(cudaMemcpyAsync(wave + starts[c], src[c], 4ull * lens[c], cudaMemcpyDeviceToDevice, s->stream), "chunk copy");
  return run_chunks(s, nullptr, wave, starts.data(), lens.data(), B);
}

// One step of any number of streams of one session (one step runs at a time).  Each stream does what a push of its samples
// (and a finish, when `final`) does alone, but the GPU work is made once for all of them:
//   1. per stream on the host: what to keep, the samples set apart during a leading silence, the window plans and room in the
//      stream's buffers;
//   2. the samples and the kernel descriptors in one pinned buffer, one host-to-device copy, one scatter launch into the
//      streams' windows, one resampling launch and one RMS launch for all windows, one download of the RMS frames and one
//      synchronise;
//   3. the slicer's decisions for each stream;
//   4. every chunk that became final, in any stream, copied next to each other and transcribed as one batch.
int streams_step(some_session* s, std::vector<StepItem>& items, Decode* dec = nullptr) {
  const int sr = s->info.sample_rate;
  StepWindows win;
  std::vector<ScatterParams> sc;
  Downmix dm;
  int64_t up_floats = 0;
  for (StepItem& it : items) {
    some_stream* st = it.st;
    const some_slicer_frames& f = st->f;
    long long keep_from, head;
    if (some_slicer_stream_keep_from(st->slicer, &keep_from, &head, nullptr)) return -1;
    // the model-rate samples a later chunk or RMS frame can still read
    const int64_t keep = std::max<int64_t>(0, std::min<int64_t>(keep_from, st->frames * f.hop_size - f.win_size / 2));
    // during a long leading silence (head > 0), the first max_sil_kept frames go apart before the window drops them (the
    // all-silent recording's one range lies there); until then the window holds everything from sample 0
    if (head == 0) {
      st->head_len = 0;
    } else if (st->head_len == 0 && keep > st->wave.first) {
      SOME_REQUIRE(st->wave.first == 0 && st->wave.len >= head, "stream: samples [0, %lld) are no longer resident",
                   (long long)head);
      if (st->head_d.ensure(4ull * head, "the stream's leading samples")) return -1;
      SOME_CUDA(cudaMemcpyAsync(st->head_d.p, st->wave.at(0), 4ull * head, cudaMemcpyDeviceToDevice, s->stream), "head copy");
      st->head_len = head;
    }
    float* dst;
    if (st->resample) {
      long long t_end, x_first;
      const double* table = table_for(s, st->rate);
      if (!table) return -1;
      if (some_resample_window_plan(st->received, 0, st->fixed, st->rate, sr, kKaiserTaps, &t_end, &x_first)) return -1;
      if (st->native.reserve(s->stream, x_first, it.n, "the stream's input")) return -1;
      dst = st->native.at(st->received);
      st->native.len += it.n, st->received += it.n;
      if (some_resample_window_plan(st->received, it.final, st->fixed, st->rate, sr, kKaiserTaps, &t_end, &x_first)) return -1;
      if (st->wave.reserve(s->stream, keep, t_end - st->fixed, "the stream's audio")) return -1;
      win.rs.push_back({st->native.at(st->native.first), st->native.first, st->received, it.final, st->wave.at(st->wave.first),
                        st->wave.first, st->fixed, t_end, st->rate, sr, table, kKaiserTaps});
      st->wave.len += t_end - st->fixed, st->fixed = t_end;
    } else {
      if (st->wave.reserve(s->stream, keep, it.n, "the stream's audio")) return -1;
      dst = st->wave.at(st->received);
      st->wave.len += it.n, st->received += it.n, st->fixed = st->received;
    }
    if (it.n && it.dev) {
      dm.push(*it.dev, it.layout, it.ready, dst);           // down-mixed straight into the window
    } else if (it.n) {
      it.up = up_floats;
      up_floats += align4(it.n);
      sc.push_back({nullptr, dst, it.n});
    }
    // the RMS frames the fixed samples complete (at the end: all of them, unless the recording is one chunk anyway)
    int64_t f_end = it.final ? frames_whole(f, st->fixed) : 0;
    if (f_end == 0) f_end = frames_within(f, st->fixed);
    it.nf = std::max<int64_t>(0, f_end - st->frames);
    if (it.nf)
      it.rms0 = win.rms({st->wave.at(st->wave.first), st->wave.first, st->wave.len, it.final ? st->fixed : -1, f.win_size,
                         f.hop_size, nullptr, st->frames, st->frames + it.nf});
  }

  // the upload: samples, then the scatter, the decode's and the windows' descriptors
  const int ks = static_cast<int>(sc.size());
  Upload up{s};
  const size_t smp_off = up.add(4ull * up_floats);
  const size_t sc_off = up.add(windows_bytes<ScatterParams>(ks));
  if (dec) dec->add(up);
  dm.add(up, static_cast<int>(dm.items.size()));
  if (win.place(s, up, "the stream upload")) return -1;
  std::vector<HostSpan> spans;
  {
    ScatterParams* ps = windows_params<ScatterParams>(up.h(sc_off), ks);
    long long* tile0 = windows_tile0(up.h(sc_off));
    int j = 0;
    for (const StepItem& it : items)
      if (it.n && !it.dev) {
        ps[j] = sc[j];
        ps[j].src = reinterpret_cast<const float*>(up.d(smp_off)) + it.up;
        tile0[j + 1] = (it.n + kScatterTile - 1) / kScatterTile;
        if (it.samples) spans.push_back({reinterpret_cast<float*>(up.h(smp_off)) + it.up, it.samples, 4ull * it.n});
        ++j;
      }
    windows_index(up.h(sc_off), ks, 0);
  }
  float* samples_d = reinterpret_cast<float*>(up.d(smp_off));
  if (dec && dec->fill(s, up, samples_d, [&](int j) { return items[j].up; })) return -1;
  if (dm.fill(s, up)) return -1;
  copy_to_pinned(*s->pool, spans, size_t(1) << 20);          // the samples, in pieces of up to 1 MB
  if (up.send("stream upload") || (dec && dec->launch(s, up))) return -1;
  if (ks) {
    const WindowsHeader& h = *reinterpret_cast<const WindowsHeader*>(up.h(sc_off));
    scatter_kernel<<<static_cast<unsigned>(h.tiles), kScatterThreads, 0, s->stream>>>(
        windows_params<ScatterParams>(up.d(sc_off), ks), windows_tile0(up.d(sc_off)), ks);
    if (check_launch("stream upload scatter")) return -1;
  }
  if (dm.launch(s, up) || win.launch(s, up)) return -1;
  SOME_CUDA(cudaStreamSynchronize(s->stream), "synchronise");   // also frees the upload buffer for the next step
  if (dec) {
    std::vector<std::pair<int, std::string>> failed;
    if (dec->check(s, up, failed)) return -1;
    for (const auto& f : failed) items[f.first].dropped = true, items[f.first].why = f.second;
  }

  // the slicer's decisions, and where each chunk that became final lies
  std::vector<const float*> src;
  std::vector<int64_t> begin, lens;
  for (StepItem& it : items) {
    some_stream* st = it.st;
    it.c0 = it.c1 = static_cast<int>(begin.size());
    if (it.dropped) continue;
    st->frames += it.nf;
    const float* rms = static_cast<const float*>(s->rms_h.p) + it.rms0;
    const int64_t* ranges = nullptr;
    int B = 0;
    if (it.final ? some_slicer_stream_finish(st->slicer, rms, static_cast<int>(it.nf), st->fixed, &ranges, &B)
                 : some_slicer_stream_feed(st->slicer, rms, static_cast<int>(it.nf), st->fixed, &ranges, &B))
      return -1;
    it.c0 = static_cast<int>(begin.size());
    if (B && ranges[0] < st->wave.first) {          // the all-silent recording's range, from the samples kept apart
      SOME_REQUIRE(B == 1 && ranges[0] == 0 && ranges[1] <= st->head_len, "stream: chunk [%lld, %lld) is not resident",
                   (long long)ranges[0], (long long)ranges[1]);
      src.push_back(static_cast<const float*>(st->head_d.p)), begin.push_back(0), lens.push_back(ranges[1]);
    } else {
      for (int i = 0; i < B; ++i) {
        SOME_REQUIRE(ranges[2 * i] >= st->wave.first && ranges[2 * i + 1] <= st->wave.first + st->wave.len,
                     "stream: chunk [%lld, %lld) is not resident ([%lld, %lld))", (long long)ranges[2 * i],
                     (long long)ranges[2 * i + 1], (long long)st->wave.first, (long long)(st->wave.first + st->wave.len));
        src.push_back(st->wave.at(ranges[2 * i]));
        begin.push_back(ranges[2 * i]), lens.push_back(std::max<int64_t>(0, ranges[2 * i + 1] - ranges[2 * i]));
      }
    }
    it.c1 = static_cast<int>(begin.size());
  }
  if (run_resident(s, src, lens)) return -1;
  for (const StepItem& it : items) take_chunks(s, it.c0, it.c1, begin.data(), lens.data(), it.out);
  return 0;
}

// The open region of a stream, [*a, *b) in model-rate samples: from the first sample a range not returned yet may begin at
// (its slicer's keep_from) to the last fixed sample.  It lies in the stream's device buffer (the buffer keeps everything from
// keep_from on, and keep_from never goes back).
int open_region(const some_stream* st, int64_t* a, int64_t* b) {
  long long from;
  if (some_slicer_stream_keep_from(st->slicer, &from, nullptr, nullptr)) return -1;
  *a = from, *b = st->fixed;
  return 0;
}

// One stream's part of a peek step: its open region, and where its notes go.
struct PeekItem {
  some_stream* st;
  some_notes* out;
  int64_t a = 0, b = 0;
  int c0 = 0, c1 = 0;           // its clip in the step's batch (none when the region is empty)
};

// A step of peeks (some_stream_peek*): the open regions of all its streams, copied from the streams' device buffers (run_resident)
// and transcribed as one batch; no stream changes.
int peeks_step(some_session* s, const std::vector<Request*>& g) {
  std::vector<const float*> src;
  std::vector<int64_t> begin, lens;
  for (Request* rq : g)
    for (PeekItem& p : *rq->peeks) {
      const some_stream* st = p.st;
      p.c0 = p.c1 = static_cast<int>(begin.size());
      if (p.b <= p.a) continue;
      SOME_REQUIRE(p.a >= st->wave.first && p.b <= st->wave.first + st->wave.len,
                   "stream: open region [%lld, %lld) is not resident ([%lld, %lld))", (long long)p.a, (long long)p.b,
                   (long long)st->wave.first, (long long)(st->wave.first + st->wave.len));
      src.push_back(st->wave.at(p.a)), begin.push_back(p.a), lens.push_back(p.b - p.a);
      p.c1 = p.c0 + 1;
    }
  if (run_resident(s, src, lens)) return -1;
  for (Request* rq : g)
    for (const PeekItem& p : *rq->peeks) take_chunks(s, p.c0, p.c1, begin.data(), lens.data(), p.out);
  return 0;
}

// Queues PCM stream items as one call (some_stream_push, some_stream_finish, some_stream_push_many).
int stream_call(some_session* s, std::vector<StepItem>& items) {
  Request rq{Request::STREAMS};
  rq.items = &items;
  for (const StepItem& it : items) {
    const some_stream* st = it.st;
    rq.samples += st->resample ? (it.n * s->info.sample_rate + st->rate - 1) / st->rate : it.n;
    rq.touches.push_back(st), rq.touches.push_back(it.out);
  }
  return submit(s, rq);
}

// One encoded stream's part of a step: its new bytes, whether the file ends there, and where its chunks go.
struct ByteItem {
  some_stream* st;
  const uint8_t* data;
  long long n;
  bool final;
  some_notes* out;
  int index;                    // in a many-call (-1: a single call)
  const char* who;              // the call, for its messages
  std::string* refusal;         // its call's first refusal
  bool live = true;             // false once refused
  int64_t up = 0, win = 0;      // its window in the bytes upload: the pending bytes that go up
  int64_t samples = 0;          // the samples it decodes in this step
  int fi = -1;                  // FLAC: its window in the step's decode
};

// A step of encoded streams (some_stream_push_bytes*, some_stream_finish):
//   1. on the host, each stream's walk consumes its bytes; their audio joins the stream's pending bytes;
//   2. the encoded-input stage (Decode) uploads the FLAC windows (the pending bytes from each stream's first unchained
//      frame) and the whole WAV or AIFF sample frames;
//   3. with FLAC streams: its scan, with the candidates down in the same synchronise as the count, then each stream's
//      resumable chain;
//   4. streams_step with the stage's decodes in front: one some_pcm_decode and one FLAC decode, mono, into the region its
//      scatter reads.
// A stream refused on its content (its walk, its chain, a decode failure, a rate or channel count the session cannot take)
// leaves the step; the others go on, and each call with a refused stream then fails with its first refusal.
int bytes_step(some_session* s, std::vector<ByteItem>& bs) {
  const int sr = s->info.sample_rate;
  auto refuse = [&](ByteItem& b) {
    b.st->failed = true, b.live = false;
    if (!b.refusal->empty()) return;
    char pre[128];
    if (b.index < 0) snprintf(pre, sizeof(pre), "%s: ", b.who);
    else snprintf(pre, sizeof(pre), "%s: stream %d: ", b.who, b.index);
    *b.refusal = std::string(pre) + some_last_error();
  };
  auto too_short = [&](ByteItem& b) {    // resampy's refusal, at the end of a file at another rate
    const some_stream* st = b.st;
    if (!b.final || !too_short_to_resample(st->received + b.samples, st->rate, sr)) return false;
    set_error("Input signal length=%lld is too small to resample from %d->%d", static_cast<long long>(st->received + b.samples),
              st->rate, sr);
    refuse(b);
    return true;
  };
  // 1. the walks
  for (ByteItem& b : bs) {
    some_stream* st = b.st;
    int known;
    long long a0, a1;
    if (st->walk->feed(b.data, b.n, b.final, &known, &a0, &a1)) {
      refuse(b);
      continue;
    }
    if (!known) continue;
    const some_audio_meta& m = st->walk->meta();
    if (st->rate == 0) {                 // this push completes the header
      if (check_format(m, sr)) {
        refuse(b);
        continue;
      }
      st->rate = m.rate, st->resample = m.rate != sr;
      st->pend_pos = st->fw.pos = m.data_offset;
    }
    if (a1 > a0 && !st->fw.done) {       // its audio bytes join the pending ones
      const std::vector<uint8_t>& held = st->walk->held_audio();
      st->pending.insert(st->pending.end(), held.begin(), held.end());
      const long long from = a0 + static_cast<long long>(held.size()), r0 = st->walk->received() - b.n;
      if (a1 > from) st->pending.insert(st->pending.end(), b.data + (from - r0), b.data + (a1 - r0));
    }
  }
  // 2. the bytes upload: each stream's pending FLAC window (from its first unchained frame) or its whole PCM sample frames
  auto flac = [](const ByteItem& b) { return b.live && b.st->rate && !pcm_container(b.st->walk->meta()); };
  std::vector<ByteWindow> ws;
  for (ByteItem& b : bs) {
    if (!b.live || !b.st->rate) continue;
    const some_audio_meta& m = b.st->walk->meta();
    b.win = static_cast<int64_t>(b.st->pending.size());
    if (pcm_container(m)) {
      const int64_t frame = static_cast<int64_t>(m.channels) * pcm_sample_bytes(m.kind);
      b.samples = b.win / frame;
      b.win = b.samples * frame;
      if (too_short(b)) continue;
    }
    ws.push_back({&m, b.st->pending.data(), b.win, &b.up});
  }
  Decode dec;
  if (dec.upload(s, ws, "the encoded streams")) return -1;
  // 3. the FLAC frames: one scan, the candidates down with the count, the chains on the host
  if (dec.nf) {
    int64_t cap = 64;
    for (const ByteItem& b : bs)
      if (flac(b)) cap += b.win / 64 + 8;
    SOME_REQUIRE(cap < (int64_t(1) << 31), "%s: too many FLAC frame candidates in one step", bs[0].who);
    if (dec.scan(s, cap, true)) return -1;
    const int n_cand = dec.n_cand;
    dec.chain.resize(std::max(n_cand, 1));
    int i = 0, k = 0;
    for (ByteItem& b : bs) {
      if (!flac(b)) continue;
      some_stream* st = b.st;
      const some_audio_meta& m = st->walk->meta();
      const int k0 = k;
      const long long base = b.up - st->pend_pos;
      if (flac_walk(dec.frames_h, n_cand, &i, base, b.up + b.win, m.frames, b.final, &st->fw, dec.chain.data(), n_cand, &k)) {
        k = k0;
        refuse(b);
        continue;
      }
      for (int j = k0; j < k; ++j) b.samples += dec.frames_h[dec.chain[j]].blocksize;
      // the bytes before the next frame are decoded (or, once the walk is done, past the recording)
      const long long keep = st->fw.done ? st->pend_pos + static_cast<long long>(st->pending.size()) : st->fw.pos;
      st->pending.erase(st->pending.begin(), st->pending.begin() + (keep - st->pend_pos));
      st->pend_pos = keep;
      if (too_short(b)) {
        k = k0;
        continue;
      }
      if (k > k0) {
        b.fi = static_cast<int>(dec.flac_of.size());
        dec.flac_of.push_back(-1);       // its step item, below
        dec.first.push_back(k);
        dec.channels.push_back(m.channels);
        dec.base.push_back(base);
      }
    }
    dec.chain.resize(k);
  }
  for (ByteItem& b : bs) {               // the PCM windows went up whole
    if (!b.live || !b.st->rate || !pcm_container(b.st->walk->meta())) continue;
    b.st->pending.erase(b.st->pending.begin(), b.st->pending.begin() + b.win);
    b.st->pend_pos += b.win;
  }
  // 4. the step: every stream whose header is complete, with its decoded samples
  std::vector<StepItem> items;
  std::vector<ByteItem*> of;
  for (ByteItem& b : bs) {
    clear(b.out);
    if (!b.live || !b.st->rate) continue;
    some_stream* st = b.st;
    const int j = static_cast<int>(items.size());
    if (b.fi >= 0) {
      dec.flac_of[b.fi] = j;
    } else if (b.samples && pcm_container(st->walk->meta())) {
      const some_audio_meta& m = st->walk->meta();
      dec.pcm.push_back(some_pcm_item{dec.bytes_d + b.up, b.samples, m.channels, m.kind, 1, 0, nullptr});
      dec.pcm_of.push_back(j);
    }
    items.push_back(StepItem{st, nullptr, b.samples, b.final, b.out});
    of.push_back(&b);
  }
  if (!items.empty() && streams_step(s, items, &dec)) return -1;
  for (size_t j = 0; j < items.size(); ++j)
    if (items[j].dropped) set_error("%s", items[j].why.c_str()), refuse(*of[j]);   // its frame failed to decode
  return 0;
}

// Queues encoded stream items as one call (some_stream_push_bytes*, some_stream_finish).
int bytes_call(some_session* s, std::vector<ByteItem>& bs) {
  Request rq{Request::BYTES};
  rq.bytes = &bs;
  for (const ByteItem& b : bs) rq.samples += b.n, rq.touches.push_back(b.st), rq.touches.push_back(b.out);
  return submit(s, rq);
}
// A step of one encoded stream (some_stream_push_bytes, some_stream_finish).
int bytes_call(some_stream* st, const void* data, long long n, bool final, some_notes* out, const char* who) {
  if (final) st->finished = true;
  std::vector<ByteItem> bs{ByteItem{st, static_cast<const uint8_t*>(data), n, final, out, -1, who}};
  return bytes_call(st->s, bs);
}

// The arguments of a many-call `who` (streams of one kind, encoded or PCM; n[i] bytes or samples at data[i]), every one
// checked before any stream changes.
template <class T>
int check_many(some_stream* const* streams, const T* const* data, const long long* n, const int* finish, int count,
               some_notes* const* out, bool encoded, const char* who) {
  some_session* s = streams[0] ? streams[0]->s : nullptr;
  std::map<const void*, int> seen, seen_notes;
  for (int i = 0; i < count; ++i) {
    const some_stream* st = streams[i];
    SOME_REQUIRE(st != nullptr, "%s: stream %d is NULL", who, i);
    SOME_REQUIRE(st->s == s, "%s: stream %d belongs to another session than stream 0", who, i);
    SOME_REQUIRE(!st->walk == !encoded, "%s: stream %d is %s", who, i,
                 encoded ? "a PCM stream (some_stream_push_many)" : "an encoded stream (some_stream_push_bytes_many)");
    const auto dup = seen.emplace(st, i);
    SOME_REQUIRE(dup.second, "%s: stream %d appears twice (also at %d)", who, i, dup.first->second);
    SOME_REQUIRE(!st->failed, "%s: stream %d was refused", who, i);     // only an encoded stream is refused
    SOME_REQUIRE(!st->finished, "%s: stream %d has finished", who, i);
    SOME_REQUIRE(n[i] >= 0 && (n[i] == 0 || data[i] != nullptr), "%s: stream %d: %lld %s at %p", who, i, n[i],
                 encoded ? "bytes" : "samples", static_cast<const void*>(data[i]));
    SOME_REQUIRE(out[i] != nullptr, "%s: stream %d: NULL notes", who, i);
    const auto shared = seen_notes.emplace(out[i], i);
    SOME_REQUIRE(shared.second, "%s: stream %d shares its some_notes with stream %d", who, i, shared.first->second);
    const int sr = s->info.sample_rate;                                 // a PCM stream's end at another rate
    SOME_REQUIRE(encoded || !(finish && finish[i]) || !too_short_to_resample(st->received + n[i], st->rate, sr),
                 "%s: stream %d: Input signal length=%lld is too small to resample from %d->%d", who, i,
                 (long long)(st->received + n[i]), st->rate, sr);
  }
  return 0;
}
}  // namespace

extern "C" int some_stream_open(some_session* s, int sample_rate, const some_slicer_params* params, some_stream** out) {
  SOME_REQUIRE(s != nullptr && out != nullptr && sample_rate > 0, "some_stream_open: bad arguments");
  *out = nullptr;
  some_slicer_frames sl;
  if (some_slicer_derive(s->info.sample_rate, params, &sl)) return -1;
  if (check_rates(sample_rate, s->info.sample_rate)) return -1;     // before any push
  some_slicer_stream* slicer;
  if (some_slicer_stream_create(&sl, &slicer)) return -1;
  some_stream* st = new some_stream();
  st->s = s, st->rate = sample_rate, st->resample = sample_rate != s->info.sample_rate;
  st->slicer = slicer, st->f = sl;
  *out = st;
  return 0;
}

extern "C" int some_stream_push(some_stream* st, const float* samples, long long n, some_notes* out) {
  SOME_REQUIRE(st != nullptr && out != nullptr && n >= 0 && (n == 0 || samples != nullptr), "some_stream_push: bad arguments");
  SOME_REQUIRE(!st->walk, "some_stream_push: an encoded stream takes bytes (some_stream_push_bytes)");
  SOME_REQUIRE(!st->finished, "some_stream_push: the stream has finished");
  std::vector<StepItem> items{StepItem{st, samples, n, false, out}};
  return stream_call(st->s, items);
}

extern "C" int some_stream_finish(some_stream* st, some_notes* out) {
  SOME_REQUIRE(st != nullptr && out != nullptr, "some_stream_finish: bad arguments");
  SOME_REQUIRE(!st->failed, "some_stream_finish: the stream was refused");
  SOME_REQUIRE(!st->finished, "some_stream_finish: the stream has finished");
  if (st->walk) return bytes_call(st, nullptr, 0, true, out, "some_stream_finish");
  const int sr = st->s->info.sample_rate;
  SOME_REQUIRE(!too_short_to_resample(st->received, st->rate, sr),
               "some_stream_finish: Input signal length=%lld is too small to resample from %d->%d", (long long)st->received,
               st->rate, sr);
  st->finished = true;
  std::vector<StepItem> items{StepItem{st, nullptr, 0, true, out}};
  return stream_call(st->s, items);
}

extern "C" int some_stream_push_many(some_stream* const* streams, const float* const* samples, const long long* n,
                                     const int* finish, int count, some_notes* const* out) {
  SOME_REQUIRE(streams != nullptr && samples != nullptr && n != nullptr && out != nullptr && count >= 0,
               "some_stream_push_many: bad arguments");
  if (count == 0) return 0;
  if (check_many(streams, samples, n, finish, count, out, false, "some_stream_push_many")) return -1;
  some_session* s = streams[0]->s;
  std::vector<StepItem> items;
  items.reserve(count);
  for (int i = 0; i < count; ++i) {
    const bool final = finish && finish[i];
    if (final) streams[i]->finished = true;
    items.push_back(StepItem{streams[i], samples[i], n[i], final, out[i]});
  }
  return stream_call(s, items);
}

extern "C" int some_stream_get_info(const some_stream* st, some_stream_info* info) {
  SOME_REQUIRE(st != nullptr && info != nullptr, "some_stream_get_info: null pointer");
  info->received = st->received, info->fixed = st->fixed, info->held = st->wave.len + st->head_len;
  return 0;
}

extern "C" int some_stream_close(some_stream* st) {
  if (st) destroy(st);
  return 0;
}

extern "C" int some_stream_open_encoded(some_session* s, const some_slicer_params* params, some_stream** out) {
  SOME_REQUIRE(s != nullptr && out != nullptr, "some_stream_open_encoded: bad arguments");
  *out = nullptr;
  some_slicer_frames sl;
  if (some_slicer_derive(s->info.sample_rate, params, &sl)) return -1;
  some_slicer_stream* slicer;
  if (some_slicer_stream_create(&sl, &slicer)) return -1;
  some_stream* st = new some_stream();
  st->s = s, st->slicer = slicer, st->f = sl;
  st->walk.reset(new AudioWalk(true));
  *out = st;
  return 0;
}

extern "C" int some_stream_push_bytes(some_stream* st, const void* data, long long n_bytes, some_notes* out) {
  SOME_REQUIRE(st != nullptr && out != nullptr && n_bytes >= 0 && (n_bytes == 0 || data != nullptr),
               "some_stream_push_bytes: bad arguments");
  SOME_REQUIRE(st->walk, "some_stream_push_bytes: a PCM stream takes samples (some_stream_push)");
  SOME_REQUIRE(!st->failed, "some_stream_push_bytes: the stream was refused");
  SOME_REQUIRE(!st->finished, "some_stream_push_bytes: the stream has finished");
  return bytes_call(st, data, n_bytes, false, out, "some_stream_push_bytes");
}

extern "C" int some_stream_push_bytes_many(some_stream* const* streams, const void* const* data, const long long* n_bytes,
                                           const int* finish, int count, some_notes* const* out) {
  SOME_REQUIRE(streams != nullptr && data != nullptr && n_bytes != nullptr && out != nullptr && count >= 0,
               "some_stream_push_bytes_many: bad arguments");
  if (count == 0) return 0;
  if (check_many(streams, data, n_bytes, finish, count, out, true, "some_stream_push_bytes_many")) return -1;
  some_session* s = streams[0]->s;
  std::vector<ByteItem> bs;
  bs.reserve(count);
  for (int i = 0; i < count; ++i) {
    const bool final = finish && finish[i];
    if (final) streams[i]->finished = true;
    bs.push_back(ByteItem{streams[i], static_cast<const uint8_t*>(data[i]), n_bytes[i], final, out[i], i,
                          "some_stream_push_bytes_many"});
  }
  return bytes_call(s, bs);
}

extern "C" int some_stream_get_meta(const some_stream* st, some_audio_meta* meta, long long* bytes_received,
                                    long long* bytes_held) {
  SOME_REQUIRE(st != nullptr && meta != nullptr, "some_stream_get_meta: null pointer");
  SOME_REQUIRE(st->walk, "some_stream_get_meta: a PCM stream has no container");
  if (st->rate) *meta = st->walk->meta();
  else *meta = some_audio_meta{};
  if (bytes_received) *bytes_received = st->walk->received();
  if (bytes_held) *bytes_held = static_cast<long long>(st->pending.size()) + st->walk->held_header();   // held_audio: in pending
  return 0;
}

namespace {
// Queues peeks of streams of one session as one call, each with its open region, whose model-rate samples size the request.
int peek_call(some_stream* const* streams, int count, some_notes* const* out) {
  std::vector<PeekItem> peeks;
  Request rq{Request::PEEKS};
  for (int i = 0; i < count; ++i) {
    PeekItem p{streams[i], out[i]};
    if (open_region(p.st, &p.a, &p.b)) return -1;
    rq.samples += std::max<int64_t>(0, p.b - p.a);
    rq.touches.push_back(p.st), rq.touches.push_back(p.out);
    peeks.push_back(p);
  }
  rq.peeks = &peeks;
  return submit(streams[0]->s, rq);
}
}  // namespace

extern "C" int some_stream_peek(some_stream* st, some_notes* out) {
  SOME_REQUIRE(st != nullptr && out != nullptr, "some_stream_peek: bad arguments");
  SOME_REQUIRE(!st->failed, "some_stream_peek: the stream was refused");
  SOME_REQUIRE(!st->finished, "some_stream_peek: the stream has finished");
  return peek_call(&st, 1, &out);
}

extern "C" int some_stream_peek_many(some_stream* const* streams, int count, some_notes* const* out) {
  const char* who = "some_stream_peek_many";
  SOME_REQUIRE(streams != nullptr && out != nullptr && count >= 0, "%s: bad arguments", who);
  if (count == 0) return 0;
  const some_session* s = streams[0] ? streams[0]->s : nullptr;
  std::map<const void*, int> seen, seen_notes;
  for (int i = 0; i < count; ++i) {
    const some_stream* st = streams[i];
    SOME_REQUIRE(st != nullptr, "%s: stream %d is NULL", who, i);
    SOME_REQUIRE(st->s == s, "%s: stream %d belongs to another session than stream 0", who, i);
    const auto dup = seen.emplace(st, i);
    SOME_REQUIRE(dup.second, "%s: stream %d appears twice (also at %d)", who, i, dup.first->second);
    SOME_REQUIRE(!st->failed, "%s: stream %d was refused", who, i);
    SOME_REQUIRE(!st->finished, "%s: stream %d has finished", who, i);
    SOME_REQUIRE(out[i] != nullptr, "%s: stream %d: NULL notes", who, i);
    const auto shared = seen_notes.emplace(out[i], i);
    SOME_REQUIRE(shared.second, "%s: stream %d shares its some_notes with stream %d", who, i, shared.first->second);
  }
  return peek_call(streams, count, out);
}

// ---------------------------------------------------------------------------------------------------- encoded files
namespace {
// Item i's message with its index in front.
std::string item_message(int i, const std::string& m) {
  return "some_session_transcribe_encoded: item " + std::to_string(i) + ": " + m;
}

// The GPU step of sliced and encoded calls (Recordings).  The encoded files' data chunks go through one Decode (with FLAC
// files: the count, then the candidates down, and some_flac_chain per file) and the sliced calls' recordings through the
// pinned staging buffer, into the recording buffer, whose Recordings are resampled, cut and transcribed after one synchronise
// (in a step of sliced calls only, when a recording is cut).  An encoded call whose file is refused after the scan (its chain,
// its length, its decode) fails with what it gives alone and leaves the step; its out[] are not written.
int recordings_step(some_session* s, const std::vector<Request*>& g) {
  const int sr = s->info.sample_rate;
  struct Ref {
    Request* rq;
    int i;
  };
  std::vector<Ref> refs;                  // every recording of the step, in call order
  for (Request* rq : g)
    for (int i = 0; i < static_cast<int>(rq->recs->size()); ++i) refs.push_back({rq, i});
  auto item = [&](const Ref& f) -> RecItem& { return (*f.rq->recs)[f.i]; };
  std::vector<ByteWindow> ws;
  std::vector<int> flac;                  // the refs of the FLAC files, in upload order
  for (int k = 0; k < static_cast<int>(refs.size()); ++k) {
    RecItem& it = item(refs[k]);
    if (it.host || it.dev) continue;
    ws.push_back({&it.m, it.bytes + it.m.data_offset, it.m.data_bytes, &it.up});
    if (!pcm_container(it.m)) flac.push_back(k);
  }
  const bool encoded = !ws.empty();
  Decode dec;
  if (encoded && dec.upload(s, ws, "the encoded files")) return -1;
  std::vector<std::vector<int32_t>> chains(flac.size());
  if (dec.nf) {
    int64_t cap = 64;
    for (int k : flac) {
      const RecItem& it = item(refs[k]);
      cap += it.m.frames ? it.m.frames / std::max(it.m.min_blocksize, 1) + 2 : it.m.data_bytes / 16 + 2;
    }
    SOME_REQUIRE(cap < (int64_t(1) << 31), "some_session_transcribe_encoded: too many FLAC frames in one call");
    if (dec.scan(s, cap, false)) return -1;
    for (size_t r = 0; r < flac.size(); ++r) {   // every file's chain first, then the lengths, as in one call
      const Ref& f = refs[flac[r]];
      RecItem& it = item(f);
      if (f.rq->rc) continue;
      const some_flac_range rec{it.up - it.m.data_offset, it.up, it.up + it.m.data_bytes, it.m.frames};
      chains[r].resize(std::max(dec.n_cand, 1));
      int64_t first[2], length = 0;
      if (some_flac_chain(dec.frames_h, dec.n_cand, &rec, 1, chains[r].data(), dec.n_cand, first, &length, nullptr)) {
        f.rq->fail(-1, item_message(f.i, some_last_error()));
        continue;
      }
      chains[r].resize(first[1]);
      it.n = length;
    }
    for (size_t r = 0; r < flac.size(); ++r) {
      const Ref& f = refs[flac[r]];
      RecItem& it = item(f);
      if (f.rq->rc) continue;
      const std::string who = "some_session_transcribe_encoded: item " + std::to_string(f.i);
      if (slice_shape(it.n, it.m.rate, sr, f.rq->sl, who.c_str(), &it.sh)) f.rq->fail(-1, some_last_error());
    }
  }
  // the recordings of the calls still in the step
  Recordings rec;
  std::vector<int> rec_of(refs.size(), -1), ref_of;
  for (int k = 0; k < static_cast<int>(refs.size()); ++k) {
    const Ref& f = refs[k];
    const RecItem& it = item(f);
    if (f.rq->rc) continue;
    const int j = static_cast<int>(rec.items.size());
    rec_of[k] = j, ref_of.push_back(k);
    rec.items.push_back({it.m.rate, it.n, it.sh, &f.rq->sl, it.out});
    if (!it.host && !it.dev && pcm_container(it.m)) {
      dec.pcm.push_back(some_pcm_item{dec.bytes_d + it.up, it.n, it.m.channels, it.m.kind, 1, 0, nullptr});
      dec.pcm_of.push_back(j);
    }
  }
  if (rec.items.empty()) return 0;
  for (size_t r = 0; r < flac.size(); ++r) {
    const int j = rec_of[flac[r]];
    if (j < 0) continue;
    const RecItem& it = item(refs[flac[r]]);
    dec.chain.insert(dec.chain.end(), chains[r].begin(), chains[r].end());
    dec.flac_of.push_back(j);
    dec.first.push_back(static_cast<int64_t>(dec.chain.size()));
    dec.channels.push_back(it.m.channels);
    dec.base.push_back(it.up - it.m.data_offset);
  }
  Upload up{s};
  if (encoded) dec.add(up);
  Downmix dm;
  dm.add(up, static_cast<int>(std::count_if(ref_of.begin(), ref_of.end(), [&](int k) { return item(refs[k]).dev != nullptr; })));
  if (rec.place(s, up)) return -1;
  std::vector<Staged> staged;
  for (size_t j = 0; j < rec.items.size(); ++j) {
    const RecItem& it = item(refs[ref_of[j]]);
    if (it.host) staged.push_back({rec.base + rec.items[j].x, it.host, it.n});
    if (it.dev) dm.push(*it.dev, it.layout, it.ready, rec.base + rec.items[j].x);
  }
  if ((!staged.empty() && upload_staged(s, staged)) ||
      (encoded && dec.fill(s, up, rec.base, [&](int j) { return rec.items[j].x; })) || dm.fill(s, up) ||
      up.send("descriptor upload") || (encoded && dec.launch(s, up)) || dm.launch(s, up) || rec.win.launch(s, up))
    return -1;
  // with a recording to cut; with device audio, so that the call returns only once its items have been read
  if (encoded || rec.win.frames || dm.k) SOME_CUDA(cudaStreamSynchronize(s->stream), "synchronise");
  if (encoded) {
    std::vector<std::pair<int, std::string>> failed;
    if (dec.check(s, up, failed)) return -1;
    for (const auto& fl : failed) {
      const Ref& f = refs[ref_of[fl.first]];
      f.rq->fail(-1, item_message(f.i, fl.second));
    }
    for (size_t j = 0; j < rec.items.size(); ++j)
      if (refs[ref_of[j]].rq->rc) rec.items[j].out = nullptr;
  }
  return rec.finish(s);
}
}  // namespace

extern "C" int some_session_transcribe_encoded(some_session* s, const some_encoded* items, int count,
                                               const some_slicer_params* params, some_notes* const* out) {
  SOME_REQUIRE(s != nullptr && items != nullptr && out != nullptr && count >= 0, "some_session_transcribe_encoded: bad arguments");
  if (count == 0) return 0;
  const int sr = s->info.sample_rate;
  some_slicer_frames sl;
  if (some_slicer_derive(sr, params, &sl)) return -1;
  // every item is checked before any GPU work
  std::vector<RecItem> its(count);
  Request rq{Request::RECORDINGS};
  rq.recs = &its, rq.sl = sl;
  std::map<const void*, int> seen_notes;
  for (int i = 0; i < count; ++i) {
    SOME_REQUIRE(items[i].data != nullptr && items[i].n_bytes > 0, "some_session_transcribe_encoded: item %d is NULL or empty", i);
    SOME_REQUIRE(out[i] != nullptr, "some_session_transcribe_encoded: item %d: NULL notes", i);
    const auto shared = seen_notes.emplace(out[i], i);
    SOME_REQUIRE(shared.second, "some_session_transcribe_encoded: item %d shares its some_notes with item %d", i,
                 shared.first->second);
    RecItem& it = its[i];
    it.bytes = static_cast<const uint8_t*>(items[i].data);
    it.out = out[i];
    if (some_audio_info(items[i].data, items[i].n_bytes, &it.m) || check_format(it.m, sr)) {
      set_error("%s", item_message(i, some_last_error()).c_str());
      return -1;
    }
    it.n = it.m.frames;
    if (pcm_container(it.m) || it.m.frames > 0) {
      const std::string who = "some_session_transcribe_encoded: item " + std::to_string(i);
      if (slice_shape(it.n, it.m.rate, sr, sl, who.c_str(), &it.sh)) return -1;
      rq.samples += it.sh.n_out;
    } else {
      rq.sized = false;                   // a FLAC file without a stated length: known only after its chain
    }
    rq.touches.push_back(out[i]);
  }
  return submit(s, rq);
}

// ---------------------------------------------------------------------------------------------------- the scheduler
namespace {
constexpr int64_t kStepSamples = SOME_SESSION_STEP_SAMPLES;

// A step of clip calls: their clips in one run_chunks, then split per call.
int clips_step(some_session* s, const std::vector<Request*>& g) {
  std::vector<const float*> clips;
  std::vector<int64_t> lens;
  for (const Request* rq : g) clips.insert(clips.end(), rq->clips, rq->clips + rq->B), lens.insert(lens.end(), rq->lens, rq->lens + rq->B);
  const int B = static_cast<int>(lens.size());
  if (run_chunks(s, clips.data(), nullptr, nullptr, lens.data(), B)) return -1;
  const std::vector<int64_t> begin(B, 0);
  int c = 0;
  for (const Request* rq : g) take_chunks(s, c, c + rq->B, begin.data(), lens.data(), rq->out), c += rq->B;
  return 0;
}

// A step of PCM stream calls, or of encoded stream calls: their items in one streams_step or bytes_step.
int streams_calls_step(some_session* s, const std::vector<Request*>& g) {
  std::vector<StepItem> items;
  for (const Request* rq : g) items.insert(items.end(), rq->items->begin(), rq->items->end());
  return streams_step(s, items);
}
int bytes_calls_step(some_session* s, const std::vector<Request*>& g) {
  std::vector<std::string> refusals(g.size());
  std::vector<ByteItem> bs;
  for (size_t k = 0; k < g.size(); ++k)
    for (ByteItem b : *g[k]->bytes) b.refusal = &refusals[k], bs.push_back(b);
  if (bytes_step(s, bs)) return -1;
  for (size_t k = 0; k < g.size(); ++k)
    if (!refusals[k].empty()) g[k]->fail(SOME_STREAM_REFUSED, refusals[k]);
  return 0;
}

// Whether a request fills a some_notes that asks for frame curves: its step then decodes curves for all its chunks, and
// each result takes them only if it asks for them.
bool wants_frames(const Request* rq) {
  auto framed = [](const auto* v) { return std::any_of(v->begin(), v->end(), [](const auto& it) { return it.out->frames; }); };
  switch (rq->kind) {
    case Request::CLIPS: return rq->out->frames;
    case Request::RECORDINGS: return framed(rq->recs);
    case Request::STREAMS: return framed(rq->items);
    case Request::BYTES: return framed(rq->bytes);
    case Request::PEEKS: return framed(rq->peeks);
  }
  return false;
}

// Runs one step on the calling thread, with the session's device current and the calls' some_set_pdl setting.  After a
// failure partway through, copies and kernels may still be queued on the session's streams: it waits for them, on every
// replica, so that the next step cannot rewrite staging or device buffers they still use; every call of the step then fails
// with the failure's message.  Returns the step's result.
int run_step(some_session* s, const std::vector<Request*>& g) {
  const int pdl = some_set_pdl(g[0]->pdl);
  int rc = -1;
  s->frames = std::any_of(g.begin(), g.end(), wants_frames);
  {
    DeviceScope scope(s->device);
    if (scope.err != cudaSuccess) {
      set_error("session: cudaSetDevice: %s", cudaGetErrorString(scope.err));
    } else {
      for (std::unique_ptr<Replica>& r : s->reps) r->chunks = r->frames = 0;
      switch (g[0]->kind) {
        case Request::CLIPS: rc = clips_step(s, g); break;
        case Request::RECORDINGS: rc = recordings_step(s, g); break;
        case Request::STREAMS: rc = streams_calls_step(s, g); break;
        case Request::BYTES: rc = bytes_calls_step(s, g); break;
        case Request::PEEKS: rc = peeks_step(s, g); break;
      }
    }
    if (rc != 0) {
      const std::string msg = some_last_error();
      for (Request* rq : g) rq->fail(-1, msg);
      for (std::unique_ptr<Replica>& r : s->reps) {
        cudaStreamSynchronize(r->copy_stream);
        cudaStreamSynchronize(r->stream);
      }
    }
  }
  some_set_pdl(pdl);
  return rc;
}

// The next step, under the session's mutex: the oldest queued call and every later call that may join it, in arrival order
// (include/some_b200.h, "Calls from several threads").  A call that cannot join keeps its place, and no later call that
// touches one of its streams or some_notes joins past it.
std::vector<Request*> take_step(some_session* s) {
  Request* first = s->queue.front();
  s->queue.pop_front();
  std::vector<Request*> g{first};
  if (!first->sized) return g;
  const int64_t bound = std::max(first->samples, kStepSamples);
  int64_t total = first->samples;
  std::set<const void*> held(first->touches.begin(), first->touches.end());
  for (auto it = s->queue.begin(); it != s->queue.end();) {
    Request* r = *it;
    bool clash = false;
    for (const void* p : r->touches) clash = clash || held.count(p) > 0;
    held.insert(r->touches.begin(), r->touches.end());
    if (clash || r->kind != first->kind || r->pdl != first->pdl || !r->sized || total + r->samples > bound) {
      ++it;
      continue;
    }
    g.push_back(r), total += r->samples;
    it = s->queue.erase(it);
  }
  return g;
}

// Queues a call and returns its result, by flat combining: while its call has not run and no step is running, the calling
// thread takes the next step (take_step) and runs it for every call in it; otherwise it waits.  Its own call's message, if
// it failed, becomes its thread's some_last_error().
int submit(some_session* s, Request& rq) {
  rq.pdl = pdl_enabled() ? 1 : 0;
  std::unique_lock<std::mutex> lock(s->mu);
  s->queue.push_back(&rq);
  ++s->stats.calls;
  while (!rq.done) {
    if (s->running) {
      s->done.wait(lock);
      continue;
    }
    const std::vector<Request*> g = take_step(s);
    s->running = true;
    ++s->stats.steps;
    s->stats.max_calls = std::max<int64_t>(s->stats.max_calls, static_cast<int64_t>(g.size()));
    lock.unlock();
    const int rc = run_step(s, g);
    lock.lock();
    if (rc == 0)
      for (size_t i = 0; i < s->reps.size(); ++i) s->load[i] = {s->reps[i]->chunks, s->reps[i]->frames};
    for (Request* r : g) r->done = true;
    s->running = false;
    s->done.notify_all();
  }
  lock.unlock();
  if (rq.rc) set_error("%s", rq.err.c_str());
  return rq.rc;
}
}  // namespace

// ---------------------------------------------------------------------------------------------------- audio on the GPU
namespace {
// An item of device audio, checked before any GPU work (prefix: the call and the item, for the message): its frames,
// channels and strides (*layout: some_downmix_layout's), and that its data is device memory of its device.
int check_device_audio(const some_device_audio& a, const std::string& prefix, int* layout) {
  const char* p = prefix.c_str();
  SOME_REQUIRE(a.frames >= 0, "%s%lld frames", p, a.frames);
  SOME_REQUIRE(a.frames == 0 || a.data != nullptr, "%sdata is NULL with %lld frames", p, a.frames);
  if (some_downmix_layout(a.channels, a.frames, a.channel_stride, a.frame_stride, layout)) {
    const std::string m = some_last_error();
    set_error("%s%s", p, m.c_str());
    return -1;
  }
  if (a.frames == 0) return 0;
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  SOME_REQUIRE(e == cudaSuccess && a.device >= 0 && a.device < n_dev, "%sno CUDA device %d", p, a.device);
  cudaPointerAttributes at{};
  e = cudaPointerGetAttributes(&at, a.data);
  if (e != cudaSuccess) cudaGetLastError();      // not a pointer the runtime knows: clear the error, refuse below
  SOME_REQUIRE(e == cudaSuccess && at.type == cudaMemoryTypeDevice && at.device == a.device,
               "%sdata %p is not device memory of device %d (%s)", p, static_cast<const void*>(a.data), a.device,
               e != cudaSuccess ? cudaGetErrorString(e)
               : at.type == cudaMemoryTypeDevice ? "it lies on another device"
               : at.type == cudaMemoryTypeManaged ? "managed memory"
               : "host memory");
  return 0;
}

// The events a call records on its items' streams (one per item with frames), destroyed when the call returns: by then the
// session's stream has passed its waits on them.
struct ReadyEvents {
  std::vector<cudaEvent_t> ev;
  ~ReadyEvents() {
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
  }
  // Records the event item `a` is read after: at this point of a.stream, on a.device.
  int record(const some_device_audio& a, const std::string& prefix, cudaEvent_t* out) {
    *out = nullptr;
    if (a.frames == 0) return 0;
    DeviceScope scope(a.device);
    cudaError_t e = scope.err;
    cudaEvent_t r = nullptr;
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&r, cudaEventDisableTiming);
    if (e == cudaSuccess) ev.push_back(r), e = cudaEventRecord(r, a.stream);
    SOME_REQUIRE(e == cudaSuccess, "%srecording an event on the item's stream: %s", prefix.c_str(), cudaGetErrorString(e));
    *out = r;
    return 0;
  }
};

// The checks of a device push to stream st, before any stream changes.
int check_push_device(const some_stream* st, const some_device_audio& a, const std::string& prefix, int* layout) {
  SOME_REQUIRE(a.sample_rate == st->rate, "%sthe audio is at %d Hz, the stream at %d Hz", prefix.c_str(), a.sample_rate,
               st->rate);
  return check_device_audio(a, prefix, layout);
}
}  // namespace

extern "C" int some_session_transcribe_device(some_session* s, const some_device_audio* items, int count,
                                              const some_slicer_params* params, some_notes* const* out) {
  const char* who = "some_session_transcribe_device";
  SOME_REQUIRE(s != nullptr && items != nullptr && out != nullptr && count >= 0, "%s: bad arguments", who);
  if (count == 0) return 0;
  const int sr = s->info.sample_rate;
  some_slicer_frames sl;
  if (some_slicer_derive(sr, params, &sl)) return -1;
  // every item is checked before any GPU work
  std::vector<RecItem> its(count);
  Request rq{Request::RECORDINGS};
  rq.recs = &its, rq.sl = sl;
  std::map<const void*, int> seen_notes;
  for (int i = 0; i < count; ++i) {
    const some_device_audio& a = items[i];
    const std::string prefix = std::string(who) + ": item " + std::to_string(i) + ": ";
    SOME_REQUIRE(out[i] != nullptr, "%sNULL notes", prefix.c_str());
    const auto shared = seen_notes.emplace(out[i], i);
    SOME_REQUIRE(shared.second, "%sshares its some_notes with item %d", prefix.c_str(), shared.first->second);
    SOME_REQUIRE(a.sample_rate > 0, "%ssample rate %d", prefix.c_str(), a.sample_rate);
    RecItem& it = its[i];
    if (check_device_audio(a, prefix, &it.layout)) return -1;
    if (check_rates(a.sample_rate, sr)) {
      const std::string m = some_last_error();
      set_error("%s%s", prefix.c_str(), m.c_str());
      return -1;
    }
    const std::string at = std::string(who) + ": item " + std::to_string(i);
    if (slice_shape(a.frames, a.sample_rate, sr, sl, at.c_str(), &it.sh)) return -1;
    it.dev = &a, it.m.rate = a.sample_rate, it.n = a.frames, it.out = out[i];
    rq.samples += it.sh.n_out;
    rq.touches.push_back(out[i]);
  }
  ReadyEvents ready;
  for (int i = 0; i < count; ++i)
    if (ready.record(items[i], std::string(who) + ": item " + std::to_string(i) + ": ", &its[i].ready)) return -1;
  return submit(s, rq);
}

extern "C" int some_stream_push_device(some_stream* st, const some_device_audio* a, some_notes* out) {
  const char* who = "some_stream_push_device";
  SOME_REQUIRE(st != nullptr && a != nullptr && out != nullptr, "%s: bad arguments", who);
  SOME_REQUIRE(!st->walk, "%s: an encoded stream takes bytes (some_stream_push_bytes)", who);
  SOME_REQUIRE(!st->finished, "%s: the stream has finished", who);
  const std::string prefix = std::string(who) + ": ";
  std::vector<StepItem> items{StepItem{st, nullptr, a->frames, false, out}};
  if (check_push_device(st, *a, prefix, &items[0].layout)) return -1;
  items[0].dev = a;
  ReadyEvents ready;
  if (ready.record(*a, prefix, &items[0].ready)) return -1;
  return stream_call(st->s, items);
}

extern "C" int some_stream_push_device_many(some_stream* const* streams, const some_device_audio* items, const int* finish,
                                            int count, some_notes* const* out) {
  const char* who = "some_stream_push_device_many";
  SOME_REQUIRE(streams != nullptr && items != nullptr && out != nullptr && count >= 0, "%s: bad arguments", who);
  if (count == 0) return 0;
  std::vector<const float*> data(count);
  std::vector<long long> n(count);
  for (int i = 0; i < count; ++i) data[i] = items[i].data, n[i] = items[i].frames;
  if (check_many(streams, data.data(), n.data(), finish, count, out, false, who)) return -1;
  std::vector<StepItem> step;
  step.reserve(count);
  for (int i = 0; i < count; ++i) {
    const bool final = finish && finish[i];
    step.push_back(StepItem{streams[i], nullptr, items[i].frames, final, out[i]});
    step.back().dev = &items[i];
    if (check_push_device(streams[i], items[i], std::string(who) + ": stream " + std::to_string(i) + ": ", &step.back().layout))
      return -1;
  }
  ReadyEvents ready;
  for (int i = 0; i < count; ++i)
    if (ready.record(items[i], std::string(who) + ": stream " + std::to_string(i) + ": ", &step[i].ready)) return -1;
  for (int i = 0; i < count; ++i)
    if (step[i].final) streams[i]->finished = true;
  return stream_call(streams[0]->s, step);
}
