// K-flac: FLAC decoding for librosa.load (libsndfile -> libFLAC), many recordings in one set of launches from slices of
// one device byte buffer.  FLAC is integer-only and lossless, so the samples are a pure function of the bitstream; the
// format is restated in oracle/flac.py (a sequential decoder and an encoder that can force every feature).
//
// some_flac_scan, four launches, no synchronisation:
//   count  one thread per FL_SCAN_BPT byte positions: how many positions of each 4 KB chunk start a frame header that is
//          syntactically valid, has a correct CRC-8 and agrees with its recording's STREAMINFO (channels, bps, block
//          size <= max).  Positions outside every recording's audio range (metadata, ID3 tags) are never candidates.
//   offsets one CTA: exclusive prefix sum of the chunk counts and the total.
//   write  the same test again; every candidate is written at its chunk's offset plus its rank inside the chunk, so the
//          list is sorted by byte position (the host finds the frame that starts at a given byte by binary search).
//   parse  one thread per candidate walks its subframes without reconstructing samples (the bit lengths of a FLAC frame
//          never depend on sample values), checks the zero padding and the CRC-16 and records the frame's byte end or,
//          for a malformed candidate, a status and the byte where the problem was found.
// The host then chains frames from each recording's first audio byte: the next frame starts where the current one ends,
// with the next frame / sample number, exactly the frames a sequential decoder walks.  A false sync pattern inside frame
// data is a candidate that is parsed and never chained.
//
// some_flac_decode, two launches over the chained frames only:
//   decode one thread per frame: subframes (CONSTANT, VERBATIM, FIXED 0-4, LPC 1-32, wasted bits), prediction with 64-bit
//          sums, stereo decorrelation, into the frame's own int32 scratch slot [channels][blocksize].
//   emit   one CTA per frame: x * 2^-(bps-1) (libsndfile's scaling, exact in float32 for bps <= 24), interleaved [n, ch] or
//          mono in numpy's order for np.mean over librosa's (channels, n) view of an [n, ch] array (mono_mean, downmix.cuh,
//          shared with the PCM decoder): channels added one after another for 2-7 channels, the pairwise tree
//          ((c0+c1)+(c2+c3))+((c4+c5)+(c6+c7)) for 8, then / channels.
//
// Every bit read is bounds-checked against the recording's byte range: reading past it yields zeros and marks the frame
// truncated, so a malformed candidate can return a status but never read outside its recording or write anywhere.
#include <stddef.h>

#include "downmix.cuh"
#include "host_common.h"

#include "../../include/some_b200.h"

static_assert(sizeof(some_flac_frame) == 40, "some_flac_frame layout (mirrored by some_b200/audio.py)");
static_assert(sizeof(some_flac_stream) == 32, "some_flac_stream layout (mirrored by some_b200/audio.py)");

namespace some {

constexpr int FL_SCAN_THREADS = 256;
constexpr int FL_SCAN_BPT = 16;                                   // byte positions per thread
constexpr int FL_SCAN_CHUNK = FL_SCAN_THREADS * FL_SCAN_BPT;
constexpr int FL_OFFS_THREADS = 1024;
constexpr int FL_FRAME_THREADS = 64;                              // parse / decode: one thread per frame
constexpr int FL_EMIT_THREADS = 256;

// ---------------------------------------------------------------------------------------------- frame header
__device__ __forceinline__ unsigned crc8_byte(unsigned crc, unsigned b) {
  crc ^= b;
#pragma unroll
  for (int k = 0; k < 8; ++k) crc = (crc & 0x80) ? ((crc << 1) ^ 0x07) & 0xFF : (crc << 1) & 0xFF;
  return crc;
}

// Index of the recording whose audio range holds byte p, or -1 (ranges sorted by audio_start, disjoint).
__device__ __forceinline__ int stream_of(const some_flac_stream* s, int n, long long p) {
  int lo = 0, hi = n - 1, r = -1;
  while (lo <= hi) {
    const int mid = (lo + hi) >> 1;
    if (s[mid].audio_start <= p) r = mid, lo = mid + 1;
    else hi = mid - 1;
  }
  return (r >= 0 && p < s[r].end) ? r : -1;
}

// Parses a frame header at byte p; true if it is a candidate.  Fills f (all fields but end / status).
__device__ __forceinline__ bool header_at(const uint8_t* data, long long n_bytes, const some_flac_stream* streams, int n_streams,
                          long long p, some_flac_frame& f) {
  if (p + 1 >= n_bytes || data[p] != 0xFF || (data[p + 1] & 0xFE) != 0xF8) return false;
  const int r = stream_of(streams, n_streams, p);
  if (r < 0) return false;
  const some_flac_stream st = streams[r];
  const long long lim = st.end;
  if (p + 6 > lim) return false;                                 // sync, codes, 1 number byte, CRC-8 at the least
  const unsigned b2 = data[p + 2], b3 = data[p + 3];
  const unsigned bs_code = b2 >> 4, sr_code = b2 & 15, ch_code = b3 >> 4, bps_code = (b3 >> 1) & 7;
  if (bs_code == 0 || sr_code == 15 || ch_code > 10 || bps_code == 3 || bps_code == 7 || (b3 & 1)) return false;
  const bool variable = data[p + 1] & 1;
  // UTF-8-like coded number: frame number (fixed blocking, up to 6 bytes / 31 bits) or sample number (up to 7 / 36 bits)
  long long q = p + 4;
  unsigned x = data[q++];
  long long number;
  int extra;
  if (x < 0x80) number = x, extra = 0;
  else if (x >= 0xC0 && x < 0xE0) number = x & 0x1F, extra = 1;
  else if (x >= 0xE0 && x < 0xF0) number = x & 0x0F, extra = 2;
  else if (x >= 0xF0 && x < 0xF8) number = x & 0x07, extra = 3;
  else if (x >= 0xF8 && x < 0xFC) number = x & 0x03, extra = 4;
  else if (x >= 0xFC && x < 0xFE) number = x & 0x01, extra = 5;
  else if (x == 0xFE && variable) number = 0, extra = 6;
  else return false;
  if (q + extra > lim) return false;
  for (int k = 0; k < extra; ++k) {
    const unsigned c = data[q++];
    if ((c & 0xC0) != 0x80) return false;
    number = (number << 6) | (c & 0x3F);
  }
  int bs;
  if (bs_code == 1) bs = 192;
  else if (bs_code <= 5) bs = 576 << (bs_code - 2);
  else if (bs_code >= 8) bs = 256 << (bs_code - 8);
  else bs = -1;                                                   // 6 / 7: explicit, read below
  const int tail = (bs_code == 6 ? 1 : bs_code == 7 ? 2 : 0) + (sr_code == 12 ? 1 : (sr_code == 13 || sr_code == 14) ? 2 : 0);
  if (q + tail + 1 > lim) return false;
  if (bs_code == 6) bs = data[q++] + 1;
  else if (bs_code == 7) bs = ((data[q] << 8) | data[q + 1]) + 1, q += 2;
  q += tail - (bs_code == 6 ? 1 : bs_code == 7 ? 2 : 0);         // the sample-rate bytes: STREAMINFO's rate is used
  unsigned crc = 0;
  for (long long k = p; k < q; ++k) crc = crc8_byte(crc, data[k]);
  if (crc != data[q]) return false;
  const int channels = ch_code < 8 ? static_cast<int>(ch_code) + 1 : 2;
  const int bps = bps_code == 0 ? st.bps : bps_code == 1 ? 8 : bps_code == 2 ? 12 : static_cast<int>(bps_code) * 4;   // 16/20/24
  if (channels != st.channels || bps != st.bps || bs > st.max_blocksize) return false;
  f.pos = p;
  f.number = number;
  f.end = 0;
  f.stream = r;
  f.blocksize = bs;
  f.header_len = static_cast<int16_t>(q + 1 - p);
  f.chan_code = static_cast<uint8_t>(ch_code);
  f.variable = variable;
  f.status = SOME_FLAC_OK;
  return true;
}

__global__ void __launch_bounds__(FL_SCAN_THREADS) flac_count_kernel(const uint8_t* data, long long n_bytes,
                                                                     const some_flac_stream* streams, int n_streams,
                                                                     int* counts) {
  __shared__ int warp_sum[FL_SCAN_THREADS / 32];
  const long long p0 = static_cast<long long>(blockIdx.x) * FL_SCAN_CHUNK + threadIdx.x * FL_SCAN_BPT;
  int c = 0;
  some_flac_frame f;
  for (int k = 0; k < FL_SCAN_BPT; ++k) c += header_at(data, n_bytes, streams, n_streams, p0 + k, f);
#pragma unroll
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < FL_SCAN_THREADS / 32; ++w) t += warp_sum[w];
    counts[blockIdx.x] = t;
  }
}

// Exclusive scan of one int per thread over the CTA; returns the CTA total through *total (all threads).
template <int kThreads>
__device__ __forceinline__ int block_exclusive_scan(int v, int* smem, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) smem[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = lane < kThreads / 32 ? smem[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += u;
    }
    if (lane < kThreads / 32) smem[lane] = w;
  }
  __syncthreads();
  const int before = (warp ? smem[warp - 1] : 0) + inc - v;
  *total = smem[kThreads / 32 - 1];
  __syncthreads();
  return before;
}

__global__ void __launch_bounds__(FL_OFFS_THREADS) flac_offsets_kernel(int* counts, int n_chunks, int* total) {
  __shared__ int smem[FL_OFFS_THREADS / 32];
  const int per = (n_chunks + FL_OFFS_THREADS - 1) / FL_OFFS_THREADS;
  const int a = min(n_chunks, static_cast<int>(threadIdx.x) * per), b = min(n_chunks, a + per);
  int s = 0;
  for (int i = a; i < b; ++i) s += counts[i];
  int all;
  int run = block_exclusive_scan<FL_OFFS_THREADS>(s, smem, &all);
  for (int i = a; i < b; ++i) {
    const int c = counts[i];
    counts[i] = run;
    run += c;
  }
  if (threadIdx.x == 0) *total = all;
}

__global__ void __launch_bounds__(FL_SCAN_THREADS, 4) flac_write_kernel(const uint8_t* data, long long n_bytes,
                                                                     const some_flac_stream* streams, int n_streams,
                                                                     const int* offsets, some_flac_frame* frames,
                                                                     int capacity) {
  __shared__ int smem[FL_SCAN_THREADS / 32];
  const long long p0 = static_cast<long long>(blockIdx.x) * FL_SCAN_CHUNK + threadIdx.x * FL_SCAN_BPT;
  unsigned hits = 0;
  some_flac_frame f;
#pragma unroll 1
  for (int k = 0; k < FL_SCAN_BPT; ++k) hits |= static_cast<unsigned>(header_at(data, n_bytes, streams, n_streams, p0 + k, f)) << k;
  int all;
  int idx = offsets[blockIdx.x] + block_exclusive_scan<FL_SCAN_THREADS>(__popc(hits), smem, &all);
#pragma unroll 1
  for (int k = 0; k < FL_SCAN_BPT; ++k) {
    if (!((hits >> k) & 1)) continue;
    header_at(data, n_bytes, streams, n_streams, p0 + k, f);
    if (idx < capacity) {
      some_flac_frame* o = frames + idx;
      o->pos = f.pos, o->number = f.number, o->end = 0, o->stream = f.stream, o->blocksize = f.blocksize;
      o->header_len = f.header_len, o->chan_code = f.chan_code, o->variable = f.variable, o->status = SOME_FLAC_OK;
    }
    ++idx;
  }
}

// ---------------------------------------------------------------------------------------------- bit reader
struct Bits {
  const uint8_t* data;
  long long byte;                 // next byte to load
  long long end;                  // first byte that may not be read
  unsigned long long cache;       // MSB-first; bits below the n valid ones are 0
  int n;
  bool over;                      // a read went past `end` (it got zeros)

  __device__ __forceinline__ void init(const uint8_t* d, long long start, long long stop) {
    data = d, byte = start, end = stop, cache = 0, n = 0, over = false;
  }
  __device__ __forceinline__ long long bitpos() const { return byte * 8 - n; }
  __device__ __forceinline__ void refill() {
    while (n <= 56 && byte < end) {
      cache |= static_cast<unsigned long long>(__ldg(data + byte)) << (56 - n);
      ++byte;
      n += 8;
    }
  }
  __device__ __forceinline__ unsigned get(int k) {              // 0 <= k <= 32
    if (k == 0) return 0;
    if (n < k) {
      refill();
      if (n < k) over = true, n = k;
    }
    const unsigned v = static_cast<unsigned>(cache >> (64 - k));
    cache = (cache << (k - 1)) << 1;
    n -= k;
    return v;
  }
  __device__ __forceinline__ int get_signed(int k) {            // 0 <= k <= 32
    if (k == 0) return 0;
    const unsigned v = get(k);
    return static_cast<int>(v << (32 - k)) >> (32 - k);
  }
  __device__ __forceinline__ unsigned unary() {                 // zeros before the next 1 (consumed)
    unsigned q = 0;
    for (;;) {
      if (n == 0) {
        refill();
        if (n == 0) {
          over = true;
          return q;
        }
      }
      const int z = cache ? __clzll(static_cast<long long>(cache)) : 64;
      if (z < n) {
        cache = (cache << z) << 1;
        n -= z + 1;
        return q + z;
      }
      q += n;
      cache = 0;
      n = 0;
    }
  }
};

// ---------------------------------------------------------------------------------------------- subframes
template <bool kStore>
__device__ int residual(Bits& br, int bs, int order, int32_t* out) {
  const unsigned method = br.get(2);
  if (method > 1) return SOME_FLAC_BAD_RESIDUAL;
  const int pbits = method ? 5 : 4;
  const unsigned esc = method ? 31u : 15u;
  const int porder = static_cast<int>(br.get(4));
  const int psize = bs >> porder;
  if ((psize << porder) != bs || psize < order) return SOME_FLAC_BAD_PARTITION;
  int i = order;
  for (int part = 0; part < (1 << porder); ++part) {
    const unsigned k = br.get(pbits);
    const int stop = (part + 1) * psize;
    if (k == esc) {
      const int w = static_cast<int>(br.get(5));
      for (; i < stop; ++i) {
        const int v = br.get_signed(w);
        if (kStore) out[i] = v;
      }
    } else {
      for (; i < stop; ++i) {
        const unsigned u = (br.unary() << k) | br.get(k);
        if (kStore) out[i] = static_cast<int>(u >> 1) ^ -static_cast<int>(u & 1);
      }
    }
    if (br.over) return SOME_FLAC_TRUNCATED;
  }
  return SOME_FLAC_OK;
}

// coef: this thread's 32 LPC coefficients (shared memory, so that the order-indexed array needs no local memory)
template <bool kStore>
__device__ int subframe(Bits& br, int bs, int sbps, int32_t* out, int* coef) {
  if (br.get(1)) return SOME_FLAC_BAD_PADDING;
  const unsigned type = br.get(6);
  int wasted = 0;
  if (br.get(1)) {
    wasted = static_cast<int>(br.unary()) + 1;
    if (wasted >= sbps) return SOME_FLAC_BAD_WASTED_BITS;
  }
  const int b = sbps - wasted;
  int rc = SOME_FLAC_OK;
  if (type == 0) {                                                 // CONSTANT
    const int v = br.get_signed(b);
    if (kStore)
      for (int i = 0; i < bs; ++i) out[i] = v;
  } else if (type == 1) {                                          // VERBATIM
    for (int i = 0; i < bs; ++i) {
      const int v = br.get_signed(b);
      if (kStore) out[i] = v;
    }
  } else if ((type & 0x38) == 0x08) {                              // FIXED
    const int order = type & 7;
    if (order > 4) return SOME_FLAC_RESERVED_SUBFRAME;
    if (order > bs) return SOME_FLAC_BAD_ORDER;
    for (int i = 0; i < order; ++i) {
      const int v = br.get_signed(b);
      if (kStore) out[i] = v;
    }
    rc = residual<kStore>(br, bs, order, out);
    if (kStore && rc == SOME_FLAC_OK) {
      for (int i = order; i < bs; ++i) {
        long long pred;
        switch (order) {
          case 0: pred = 0; break;
          case 1: pred = out[i - 1]; break;
          case 2: pred = 2ll * out[i - 1] - out[i - 2]; break;
          case 3: pred = 3ll * out[i - 1] - 3ll * out[i - 2] + out[i - 3]; break;
          default: pred = 4ll * out[i - 1] - 6ll * out[i - 2] + 4ll * out[i - 3] - out[i - 4]; break;
        }
        out[i] = static_cast<int>(static_cast<long long>(out[i]) + pred);
      }
    }
  } else if (type & 0x20) {                                        // LPC
    const int order = static_cast<int>(type & 31) + 1;
    if (order > bs) return SOME_FLAC_BAD_ORDER;
    for (int i = 0; i < order; ++i) {
      const int v = br.get_signed(b);
      if (kStore) out[i] = v;
    }
    const int precision = static_cast<int>(br.get(4)) + 1;
    if (precision == 16) return SOME_FLAC_BAD_LPC;
    const int shift = br.get_signed(5);
    if (shift < 0) return SOME_FLAC_BAD_LPC;
    for (int j = 0; j < order; ++j) {
      const int c = br.get_signed(precision);
      if (kStore) coef[j * FL_FRAME_THREADS] = c;
    }
    rc = residual<kStore>(br, bs, order, out);
    if (kStore && rc == SOME_FLAC_OK) {
      for (int i = order; i < bs; ++i) {
        long long sum = 0;
        for (int j = 0; j < order; ++j) sum += static_cast<long long>(coef[j * FL_FRAME_THREADS]) * out[i - 1 - j];
        out[i] = static_cast<int>(static_cast<long long>(out[i]) + (sum >> shift));
      }
    }
  } else {
    return SOME_FLAC_RESERVED_SUBFRAME;
  }
  if (rc != SOME_FLAC_OK) return rc;
  if (br.over) return SOME_FLAC_TRUNCATED;
  if (kStore && wasted)
    for (int i = 0; i < bs; ++i) out[i] = static_cast<int>(static_cast<unsigned>(out[i]) << wasted);
  return SOME_FLAC_OK;
}

// Walks one frame (header already parsed into f).  kStore: writes the decoded, decorrelated samples to out
// [channels][blocksize].  Returns the status; *end = one past the CRC-16 (OK) or the byte where the problem was found.
template <bool kStore>
__device__ int walk_frame(const uint8_t* data, const some_flac_stream& st, const some_flac_frame& f, const uint16_t* crc16,
                          int32_t* out, int* coef, long long* end) {
  Bits br;
  br.init(data, f.pos + f.header_len, st.end);
  const int bs = f.blocksize;
  int rc = SOME_FLAC_OK;
  for (int c = 0; c < st.channels && rc == SOME_FLAC_OK; ++c) {
    const bool side = (f.chan_code == 8 && c == 1) || (f.chan_code == 9 && c == 0) || (f.chan_code == 10 && c == 1);
    rc = subframe<kStore>(br, bs, st.bps + side, out + static_cast<long long>(c) * bs, coef);
  }
  if (rc == SOME_FLAC_OK) {
    if (br.get((8 - static_cast<int>(br.bitpos() & 7)) & 7)) rc = SOME_FLAC_BAD_PADDING;
    const unsigned want = br.get(16);
    if (br.over) rc = SOME_FLAC_TRUNCATED;
    if (rc == SOME_FLAC_OK && !kStore) {
      const long long stop = br.bitpos() >> 3;
      unsigned crc = 0;
      for (long long k = f.pos; k < stop - 2; ++k) crc = ((crc << 8) ^ crc16[((crc >> 8) ^ __ldg(data + k)) & 0xFF]) & 0xFFFF;
      if (crc != want) rc = SOME_FLAC_BAD_CRC16;
    }
  }
  *end = min(br.bitpos() >> 3, static_cast<long long>(st.end));
  if (kStore && rc == SOME_FLAC_OK && st.channels == 2 && f.chan_code >= 8) {
    int32_t* a = out;
    int32_t* b = out + bs;
    for (int i = 0; i < bs; ++i) {
      const int x = a[i], y = b[i];
      if (f.chan_code == 8) {                                        // left / side
        b[i] = x - y;
      } else if (f.chan_code == 9) {                                 // side / right
        a[i] = x + y;
      } else {                                                       // mid / side
        const int m = static_cast<int>((static_cast<unsigned>(x) << 1) | (static_cast<unsigned>(y) & 1u));
        a[i] = (m + y) >> 1;
        b[i] = (m - y) >> 1;
      }
    }
  }
  return rc;
}

__device__ __forceinline__ void fill_crc16(uint16_t* t) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    unsigned c = static_cast<unsigned>(i) << 8;
    for (int k = 0; k < 8; ++k) c = (c & 0x8000) ? ((c << 1) ^ 0x8005) : (c << 1);
    t[i] = static_cast<uint16_t>(c & 0xFFFF);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(FL_FRAME_THREADS) flac_parse_kernel(const uint8_t* data, const some_flac_stream* streams,
                                                                      some_flac_frame* frames, const int* count, int capacity) {
  __shared__ uint16_t crc16[256];
  fill_crc16(crc16);
  const int i = blockIdx.x * FL_FRAME_THREADS + threadIdx.x;
  if (i >= min(*count, capacity)) return;
  some_flac_frame f = frames[i];
  long long end;
  const int rc = walk_frame<false>(data, streams[f.stream], f, crc16, nullptr, nullptr, &end);
  frames[i].end = end;
  frames[i].status = rc;
}

__global__ void __launch_bounds__(FL_FRAME_THREADS) flac_decode_kernel(const uint8_t* data, const some_flac_stream* streams,
                                                                       const some_flac_frame* frames, const int32_t* chain,
                                                                       const int64_t* scratch_off, int n_chain,
                                                                       int32_t* scratch, int* status, int* failed) {
  __shared__ int coef[32 * FL_FRAME_THREADS];                      // [j][thread]: conflict-free
  const int k = blockIdx.x * FL_FRAME_THREADS + threadIdx.x;
  if (k >= n_chain) return;
  const some_flac_frame f = frames[chain[k]];
  long long end;
  const int rc = walk_frame<true>(data, streams[f.stream], f, nullptr, scratch + scratch_off[k], coef + threadIdx.x, &end);
  if (rc != SOME_FLAC_OK) {                                        // a chained frame parsed OK: never expected
    atomicCAS(status, 0, rc);
    if (failed) atomicMin(failed, k);
  }
}

__global__ void __launch_bounds__(FL_EMIT_THREADS) flac_emit_kernel(const some_flac_stream* streams,
                                                                    const some_flac_frame* frames, const int32_t* chain,
                                                                    const int64_t* scratch_off, const int64_t* out_off,
                                                                    const int32_t* scratch, float* out, int mono) {
  const int k = blockIdx.x;
  const some_flac_frame f = frames[chain[k]];
  const int ch = streams[f.stream].channels, bs = f.blocksize;
  const float scale = __int_as_float((127 - (streams[f.stream].bps - 1)) << 23);     // 2^-(bps-1), exact
  const int32_t* s = scratch + scratch_off[k];
  float* y = out + out_off[k] * (mono ? 1 : ch);
  for (int i = threadIdx.x; i < bs; i += FL_EMIT_THREADS) {
    if (!mono) {
      for (int c = 0; c < ch; ++c) y[static_cast<long long>(i) * ch + c] = __fmul_rn(static_cast<float>(s[c * bs + i]), scale);
      continue;
    }
    y[i] = mono_mean(ch, [&](int c) { return __fmul_rn(static_cast<float>(s[c * bs + i]), scale); });
  }
}

}  // namespace some

using namespace some;

extern "C" uint64_t some_flac_scan_workspace_bytes(long long n_bytes) {
  const long long chunks = (n_bytes + FL_SCAN_CHUNK - 1) / FL_SCAN_CHUNK;
  return static_cast<uint64_t>(chunks > 0 ? chunks : 1) * sizeof(int);
}

extern "C" int some_flac_scan(const uint8_t* data, long long n_bytes, const some_flac_stream* streams, int n_streams,
                              some_flac_frame* frames, int capacity, int* count, void* workspace, cudaStream_t stream) {
  SOME_REQUIRE(data && streams && count && workspace && (frames || capacity == 0), "some_flac_scan: null pointer");
  SOME_REQUIRE(n_bytes >= 0 && n_bytes < (1ll << 31), "some_flac_scan: %lld bytes (at most 2^31 - 1 per call)", n_bytes);
  SOME_REQUIRE(n_streams >= 0 && capacity >= 0, "some_flac_scan: bad sizes (%d streams, capacity %d)", n_streams, capacity);
  const int chunks = static_cast<int>((n_bytes + FL_SCAN_CHUNK - 1) / FL_SCAN_CHUNK);
  if (chunks == 0 || n_streams == 0) {
    cudaError_t e = cudaMemsetAsync(count, 0, sizeof(int), stream);
    SOME_REQUIRE(e == cudaSuccess, "some_flac_scan: %s", cudaGetErrorString(e));
    return 0;
  }
  int* counts = static_cast<int*>(workspace);
  flac_count_kernel<<<chunks, FL_SCAN_THREADS, 0, stream>>>(data, n_bytes, streams, n_streams, counts);
  flac_offsets_kernel<<<1, FL_OFFS_THREADS, 0, stream>>>(counts, chunks, count);
  flac_write_kernel<<<chunks, FL_SCAN_THREADS, 0, stream>>>(data, n_bytes, streams, n_streams, counts, frames, capacity);
  if (capacity > 0)
    flac_parse_kernel<<<(capacity + FL_FRAME_THREADS - 1) / FL_FRAME_THREADS, FL_FRAME_THREADS, 0, stream>>>(
        data, streams, frames, count, capacity);
  return check_launch("some_flac_scan");
}

int some::flac_decode_chain(const uint8_t* data, const some_flac_stream* streams, const some_flac_frame* frames,
                            const int32_t* chain, const int64_t* scratch_off, const int64_t* out_off, int n_chain,
                            int32_t* scratch, float* out, int mono, int* status, int* failed, cudaStream_t stream) {
  SOME_REQUIRE(data && streams && frames && chain && scratch_off && out_off && scratch && out && status,
               "some_flac_decode: null pointer");
  SOME_REQUIRE(n_chain >= 0, "some_flac_decode: %d frames", n_chain);
  if (n_chain == 0) return 0;
  flac_decode_kernel<<<(n_chain + FL_FRAME_THREADS - 1) / FL_FRAME_THREADS, FL_FRAME_THREADS, 0, stream>>>(
      data, streams, frames, chain, scratch_off, n_chain, scratch, status, failed);
  flac_emit_kernel<<<n_chain, FL_EMIT_THREADS, 0, stream>>>(streams, frames, chain, scratch_off, out_off, scratch, out, mono);
  return check_launch("some_flac_decode");
}

extern "C" int some_flac_decode(const uint8_t* data, const some_flac_stream* streams, const some_flac_frame* frames,
                                const int32_t* chain, const int64_t* scratch_off, const int64_t* out_off, int n_chain,
                                int32_t* scratch, float* out, int mono, int* status, cudaStream_t stream) {
  return flac_decode_chain(data, streams, frames, chain, scratch_off, out_off, n_chain, scratch, out, mono, status, nullptr,
                           stream);
}
