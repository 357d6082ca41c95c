// Host-only helpers of the encoded-file path (no CUDA call): container metadata (some_audio_info), the FLAC frame chain
// (some_flac_chain) and Standard MIDI File bytes (some_midi_write, some_notes_midi).
//
// some_audio_info restates what some_b200.audio.load accepts, except integer PCM in 5-8 byte containers (scipy: int64,
// x / 2^63) and 1-8 bit PCM in wider containers, which it refuses: RIFF/WAVE exactly as scipy.io.wavfile.read walks it (the
// chunk loop bounded by the RIFF size, the pad byte of odd chunks, a data chunk cut short by the end of the file), and FLAC
// with audio.parse_flac's metadata-block rules.  Its refusals carry the Python reason and a byte offset.
// some_flac_chain is the one copy of the walk FlacBatch used to do in Python; both the Python and the session's paths call it.
// some_midi_write is some_b200.midi.build_midi_file(...).to_bytes(), tick for tick.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "host_common.h"

#include "../../include/some_b200.h"

using namespace some;

namespace {

uint32_t le32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | (static_cast<uint32_t>(p[3]) << 24); }
uint16_t le16(const uint8_t* p) { return static_cast<uint16_t>(p[0] | (p[1] << 8)); }

// audio._id3_size: 10 + the syncsafe size (+ 10 with a footer), 0 without a tag.
long long id3_size(const uint8_t* d, long long n) {
  if (n < 10 || memcmp(d, "ID3", 3) != 0) return 0;
  const long long size = (d[6] & 0x7F) << 21 | (d[7] & 0x7F) << 14 | (d[8] & 0x7F) << 7 | (d[9] & 0x7F);
  return 10 + size + ((d[5] & 0x10) ? 10 : 0);
}

// audio.parse_flac
int flac_info(const uint8_t* d, long long n, long long off, some_audio_meta* m) {
  long long p = off + 4;
  bool first = true;
  int min_bs = 0, max_bs = 0, rate = 0, channels = 0, bps = 0;
  long long length = 0;
  for (;;) {
    SOME_REQUIRE(p + 4 <= n, "FLAC metadata block header truncated at byte offset %lld", p);
    const int last = d[p] >> 7, kind = d[p] & 0x7F;
    const long long size = (static_cast<long long>(d[p + 1]) << 16) | (d[p + 2] << 8) | d[p + 3];
    SOME_REQUIRE(!(first && (kind != 0 || size != 34)),
                 "FLAC stream does not start with a 34-byte STREAMINFO block (type %d, %lld bytes at byte offset %lld)", kind,
                 size, p);
    SOME_REQUIRE(first || (kind != 0 && kind != 127), "%s FLAC metadata block at byte offset %lld",
                 kind == 0 ? "second STREAMINFO" : "invalid", p);
    SOME_REQUIRE(p + 4 + size <= n, "FLAC metadata block truncated at byte offset %lld", p);
    if (first) {
      const uint8_t* b = d + p + 4;
      min_bs = (b[0] << 8) | b[1];
      max_bs = (b[2] << 8) | b[3];
      rate = (b[10] << 12) | (b[11] << 4) | (b[12] >> 4);
      channels = ((b[12] >> 1) & 7) + 1;
      bps = (((b[12] & 1) << 4) | (b[13] >> 4)) + 1;
      length = (static_cast<long long>(b[13] & 15) << 32) | (static_cast<long long>(b[14]) << 24) | (b[15] << 16) |
               (b[16] << 8) | b[17];
      first = false;
    }
    p += 4 + size;
    if (last) break;
  }
  SOME_REQUIRE(bps <= 24,
               "FLAC stream of %d bits per sample (at byte offset %lld); only up to 24 bits are decoded (libsndfile's float "
               "scaling is exact up to 24 bits)",
               bps, off + 8);
  SOME_REQUIRE(rate != 0 && max_bs != 0, "invalid FLAC STREAMINFO (sample rate %d, max block size %d) at byte offset %lld", rate,
               max_bs, off + 8);
  m->container = SOME_AUDIO_FLAC;
  m->rate = rate, m->channels = channels, m->bits = bps, m->kind = 0;
  m->min_blocksize = min_bs, m->max_blocksize = max_bs;
  m->frames = length;
  m->data_offset = p;
  m->data_bytes = n - p;
  return 0;
}

// The container named in audio.decode_wav's refusal of a file that is not RIFF/WAVE.
std::string not_wave_kind(const uint8_t* d, long long n) {
  static const struct {
    const char* magic;
    const char* name;
  } formats[] = {{"fLaC", "FLAC"},   {"OggS", "Ogg"},   {"ID3", "MP3 (ID3 tag)"},    {"FORM", "AIFF/IFF"},
                 {"RIFX", "big-endian RIFX"}, {"RF64", "RF64"}, {"caff", "Core Audio (CAF)"}, {".snd", "Sun/NeXT AU"}};
  const long long h = n < 12 ? n : 12;
  for (const auto& f : formats) {
    const long long k = static_cast<long long>(strlen(f.magic));
    if (h >= k && memcmp(d, f.magic, k) == 0) return f.name;
  }
  if (h >= 2 && d[0] == 0xFF && (d[1] & 0xE0) == 0xE0) return "MPEG audio (MP3)";
  std::string s = "unrecognised header";
  char hex[4];
  for (long long i = 0; i < h; ++i) snprintf(hex, sizeof(hex), " %02x", d[i]), s += hex;
  return s;
}

// scipy.io.wavfile.read's walk over a RIFF/WAVE file (little-endian RIFF only: audio.decode_wav refuses the rest first).
// `pos` follows the file position scipy's reads and seeks leave, so the chunk loop ends where scipy's does.
int wav_info(const uint8_t* d, long long n, some_audio_meta* m) {
  const long long file_size = static_cast<long long>(le32(d + 4)) + 8;
  long long pos = 12;
  bool have_fmt = false, have_data = false;
  int tag = 0, channels = 0, rate = 0, block_align = 0, bits = 0;
  int d_kind = 0, d_channels = 0, d_bits = 0;
  long long d_frames = 0, d_offset = 0, d_bytes = 0;
  while (pos < file_size) {
    const long long p = pos;
    if (p >= n) {
      SOME_REQUIRE(have_data, "RIFF/WAVE: Unexpected end of file. (at byte offset %lld)", p);
      break;
    }
    if (n - p < 4) {
      SOME_REQUIRE(have_fmt && have_data, "RIFF/WAVE: Incomplete chunk ID (at byte offset %lld)", p);
      break;                                                     // scipy warns and stops at the end of the file
    }
    const uint8_t* id = d + p;
    const bool is_fmt = memcmp(id, "fmt ", 4) == 0, is_data = memcmp(id, "data", 4) == 0;
    if (!is_fmt && !is_data) {                                   // fact, LIST, JUNK, Fake and unknown chunks: skipped
      if (n - p == 4) {
        pos = n;
        continue;
      }
      SOME_REQUIRE(n - p >= 8, "RIFF/WAVE: '%.4s' chunk size truncated at byte offset %lld", id, p);
      const long long size = le32(d + p + 4);
      pos = p + 8 + size + (size & 1);
      continue;
    }
    SOME_REQUIRE(n - p >= 8, "RIFF/WAVE: '%.4s' chunk size truncated at byte offset %lld", id, p);
    const long long size = le32(d + p + 4);
    if (is_fmt) {
      SOME_REQUIRE(size >= 16, "RIFF/WAVE: Binary structure of wave file is not compliant (fmt chunk of %lld bytes at byte offset "
                   "%lld)", size, p);
      SOME_REQUIRE(n - p >= 24, "RIFF/WAVE: fmt chunk truncated at byte offset %lld", p);
      const uint8_t* b = d + p + 8;
      tag = le16(b), channels = le16(b + 2), rate = static_cast<int>(le32(b + 4)), block_align = le16(b + 12);
      bits = le16(b + 14);
      const uint32_t byte_rate = le32(b + 8);
      if (tag == 0xFFFE && size >= 18) {
        SOME_REQUIRE(n - p >= 26, "RIFF/WAVE: fmt chunk truncated at byte offset %lld", p);
        const int ext = le16(b + 16);
        SOME_REQUIRE(ext >= 22, "RIFF/WAVE: Binary structure of wave file is not compliant (extension of %d bytes at byte "
                     "offset %lld)", ext, p);
        static const uint8_t tail[12] = {0x00, 0x00, 0x10, 0x00, 0x80, 0x00, 0x00, 0xAA, 0x00, 0x38, 0x9B, 0x71};
        if (n - p >= 8 + 18 + 22 && memcmp(b + 18 + 6 + 4, tail, 12) == 0) tag = static_cast<int>(le32(b + 18 + 6));
      }
      SOME_REQUIRE(tag == 1 || tag == 3, "RIFF/WAVE: Unknown wave file format: %#06x. Supported formats: PCM, IEEE_FLOAT (fmt chunk "
                   "at byte offset %lld)", tag, p);
      pos = std::min(p + 8 + size, n) + (size & 1);
      SOME_REQUIRE(tag != 1 || byte_rate == static_cast<uint32_t>(rate) * static_cast<uint32_t>(block_align),
                   "RIFF/WAVE: WAV header is invalid: nAvgBytesPerSec must equal product of nSamplesPerSec and nBlockAlign, but "
                   "file has nSamplesPerSec = %d, nBlockAlign = %d, and nAvgBytesPerSec = %u (fmt chunk at byte offset %lld)",
                   rate, block_align, byte_rate, p);
      have_fmt = true;
      continue;
    }
    // data
    SOME_REQUIRE(have_fmt, "RIFF/WAVE: No fmt chunk before data (data chunk at byte offset %lld)", p);
    SOME_REQUIRE(channels > 0 && block_align / channels > 0,
                 "RIFF/WAVE: %d channels in blocks of %d bytes (data chunk at byte offset %lld)", channels, block_align, p);
    const int bps = block_align / channels;                     // scipy's container size
    int kind = 0, isz = bps;
    if (tag == 1) {
      SOME_REQUIRE(bits <= 64, "RIFF/WAVE: Unsupported bit depth: the WAV file has %d-bit integer data. (data chunk at byte "
                   "offset %lld)", bits, p);
      if (bits >= 1 && bits <= 8) kind = bps == 1 ? SOME_PCM_U8 : 0, isz = 1;
      else kind = bps == 2 ? SOME_PCM_S16 : bps == 3 ? SOME_PCM_S24 : bps == 4 ? SOME_PCM_S32 : 0;
      SOME_REQUIRE(kind, "RIFF/WAVE: %d-bit PCM in %d-byte containers is not read (u8, s16, s24 and s32 are; data chunk at "
                   "byte offset %lld)", bits, bps, p);
    } else {
      SOME_REQUIRE(bits == 32 || bits == 64, "RIFF/WAVE: Unsupported bit depth: the WAV file has %d-bit floating-point data. "
                   "(data chunk at byte offset %lld)", bits, p);
      kind = bps == 4 ? SOME_PCM_F32 : bps == 8 ? SOME_PCM_F64 : 0;
      SOME_REQUIRE(kind, "RIFF/WAVE: %d-bit float in %d-byte containers (data chunk at byte offset %lld)", bits, bps, p);
    }
    const long long avail = n - (p + 8);
    long long samples, consumed;
    if (kind == SOME_PCM_S24) {                                  // read as raw bytes, then regrouped by three
      consumed = std::min(size, avail);
      SOME_REQUIRE(consumed % 3 == 0, "RIFF/WAVE: %lld bytes of 24-bit samples are not a whole number of samples (data chunk at "
                   "byte offset %lld)", consumed, p);
      samples = consumed / 3;
    } else {
      const long long want = size / bps;                        // items of isz bytes (u8: one byte each)
      samples = std::min(want, avail / isz);
      consumed = std::min(want * isz, avail);
    }
    SOME_REQUIRE(channels == 1 || samples % channels == 0,
                 "RIFF/WAVE: %lld samples do not fill whole frames of %d channels (data chunk at byte offset %lld)", samples,
                 channels, p);
    have_data = true;
    d_kind = kind, d_channels = channels, d_bits = bits;
    d_frames = samples / channels, d_offset = p + 8, d_bytes = samples * isz;
    pos = p + 8 + consumed + (size & 1);
  }
  SOME_REQUIRE(have_fmt, "RIFF/WAVE: no fmt chunk");
  SOME_REQUIRE(have_data, "RIFF/WAVE: no data chunk");
  m->container = SOME_AUDIO_WAV;
  m->rate = rate, m->channels = d_channels, m->bits = d_bits, m->kind = d_kind;
  m->min_blocksize = 0, m->max_blocksize = 0;
  m->frames = d_frames, m->data_offset = d_offset, m->data_bytes = d_bytes;
  return 0;
}

const char* flac_reason(int status, char* buf, size_t cap) {
  static const char* reasons[] = {nullptr,
                                  "truncated frame",
                                  "CRC-16 mismatch",
                                  "non-zero padding bits",
                                  "reserved subframe type",
                                  "invalid wasted-bits count",
                                  "predictor order larger than the block",
                                  "invalid LPC precision or shift",
                                  "reserved residual coding method",
                                  "invalid partition order"};
  if (status >= 1 && status <= 9) return reasons[status];
  snprintf(buf, cap, "%d", status);
  return buf;
}

// Variable-length quantity of a MIDI delta time.
void put_varlen(std::vector<uint8_t>& o, uint64_t v) {
  uint8_t tmp[10];
  int k = 0;
  tmp[k++] = v & 0x7F;
  for (v >>= 7; v; v >>= 7) tmp[k++] = static_cast<uint8_t>((v & 0x7F) | 0x80);
  while (k) o.push_back(tmp[--k]);
}

}  // namespace

extern "C" int some_audio_info(const void* data, long long n_bytes, some_audio_meta* out) {
  SOME_REQUIRE(out != nullptr && n_bytes >= 0 && (data != nullptr || n_bytes == 0), "some_audio_info: bad arguments");
  const uint8_t* d = static_cast<const uint8_t*>(data);
  some_audio_meta m{};
  const long long off = id3_size(d, n_bytes);
  if (off + 4 <= n_bytes && memcmp(d + off, "fLaC", 4) == 0) {
    if (flac_info(d, n_bytes, off, &m)) return -1;
  } else {
    SOME_REQUIRE(n_bytes >= 12 && memcmp(d, "RIFF", 4) == 0 && memcmp(d + 8, "WAVE", 4) == 0,
                 "not a RIFF/WAVE file (%s); some_b200.audio reads WAV files only", not_wave_kind(d, n_bytes).c_str());
    if (wav_info(d, n_bytes, &m)) return -1;
  }
  *out = m;
  return 0;
}

extern "C" int some_flac_chain(const some_flac_frame* frames, int n_frames, const some_flac_range* recs, int n_recs, int32_t* chain,
                               int capacity, int64_t* first, int64_t* lengths, int* failed) {
  SOME_REQUIRE((frames || n_frames == 0) && (recs || n_recs == 0) && (chain || capacity == 0) && first && lengths &&
                   n_frames >= 0 && n_recs >= 0 && capacity >= 0,
               "some_flac_chain: bad arguments");
  if (failed) *failed = -1;
  int i = 0, k = 0;
  first[0] = 0;
  char buf[16];
  for (int r = 0; r < n_recs; ++r) {
    const long long base = recs[r].base, stop = recs[r].end, total = recs[r].length;
    long long p = recs[r].audio_start, got = 0, count = 0;
    int strategy = -1;
    auto fail = [&]() {
      if (failed) *failed = r;
      return -1;
    };
    while (!(total && got == total) && !(!total && p == stop)) {
      if (p >= stop) {
        set_error("FLAC stream ends at byte offset %lld after %lld of %lld samples", p - base, got, total);
        return fail();
      }
      while (i < n_frames && frames[i].pos < p) ++i;
      if (i >= n_frames || frames[i].pos != p) {
        set_error("no valid FLAC frame header (sync, reserved code, CRC-8 or STREAMINFO mismatch) at byte offset %lld", p - base);
        return fail();
      }
      const some_flac_frame& f = frames[i];
      if (f.status) {
        set_error("FLAC frame at byte offset %lld: %s (at byte offset %lld)", p - base, flac_reason(f.status, buf, sizeof(buf)),
                  static_cast<long long>(f.end) - base);
        return fail();
      }
      if (strategy < 0) strategy = f.variable;
      const long long want = f.variable ? got : count;
      if (f.variable != strategy || f.number != want) {
        set_error("FLAC frame at byte offset %lld: %s number %lld, expected %lld (gap, overlap or changed blocking strategy)",
                  p - base, f.variable ? "sample" : "frame", static_cast<long long>(f.number), want);
        return fail();
      }
      got += f.blocksize;
      if (total && got > total) {
        set_error("FLAC frame at byte offset %lld decodes past the %lld samples STREAMINFO states", p - base, total);
        return fail();
      }
      if (k >= capacity) {
        set_error("some_flac_chain: more than %d chained frames", capacity);
        return fail();
      }
      chain[k++] = i;
      ++count;
      p = f.end;
    }
    first[r + 1] = k;
    lengths[r] = got;
  }
  return 0;
}

extern "C" int some_midi_write(int n_chunks, const double* offsets, const int32_t* counts, const float* note_midi,
                               const int32_t* note_dur, const uint8_t* note_rest, double timestep, double tempo, uint8_t* buf,
                               size_t capacity, size_t* size) {
  SOME_REQUIRE(n_chunks >= 0 && size != nullptr && (n_chunks == 0 || (offsets && counts)) && (buf || capacity == 0),
               "some_midi_write: bad arguments");
  const double us = rint(60.0 * 1000000.0 / tempo);               // midi.bpm2tempo: int(round(60e6 / bpm))
  SOME_REQUIRE(us >= 0 && us < 16777216.0, "some_midi_write: tempo %g bpm is %.0f microseconds per beat, which does not fit the 24 "
               "bits of set_tempo", tempo, us);
  const double tps = tempo * 8;                                    // ticks per second at 480 ticks per beat
  std::vector<uint8_t> trk;
  put_varlen(trk, 0);
  trk.insert(trk.end(), {0xFF, 0x51, 0x03});
  const uint32_t t = static_cast<uint32_t>(us);
  trk.insert(trk.end(), {static_cast<uint8_t>(t >> 16), static_cast<uint8_t>(t >> 8), static_cast<uint8_t>(t)});
  long long last = 0;
  int64_t a = 0;
  for (int c = 0; c < n_chunks; ++c) {
    SOME_REQUIRE(counts[c] >= 0, "some_midi_write: chunk %d has %d notes", c, counts[c]);
    SOME_REQUIRE(counts[c] == 0 || (note_midi && note_dur && note_rest), "some_midi_write: null note arrays");
    const long long t0 = static_cast<long long>(rint(offsets[c] * tps));
    const bool has_limit = c + 1 < n_chunks;
    const long long limit = has_limit ? static_cast<long long>(rint(offsets[c + 1] * tps)) : 0;
    long long start = t0, prev_end = 0;
    double acc = 0.0;                                              // np.cumsum of the durations in seconds
    for (int j = 0; j < counts[c]; ++j, ++a) {
      acc += static_cast<double>(note_dur[a]) * timestep;
      const long long e = static_cast<long long>(rint(acc * tps));
      const long long len = e - prev_end;
      prev_end = e;
      long long end = start + len;
      if (has_limit && end > limit) end = limit;
      if (start < end && !note_rest[a]) {
        const float p = rintf(note_midi[a]);
        SOME_REQUIRE(p >= 0.f && p <= 127.f, "some_midi_write: attribute must be in range 0..127: note=%.0f (chunk %d, note %d)",
                     static_cast<double>(p), c, j);
        const long long delta = start - last;
        SOME_REQUIRE(delta >= 0, "some_midi_write: message time must be non-negative in a MIDI file (chunk %d, note %d)", c, j);
        const uint8_t note = static_cast<uint8_t>(p);
        put_varlen(trk, static_cast<uint64_t>(delta));
        trk.insert(trk.end(), {0x90, note, 64});
        put_varlen(trk, static_cast<uint64_t>(end - start));
        trk.insert(trk.end(), {0x80, note, 64});
        last = end;
      }
      start = end;
    }
  }
  trk.insert(trk.end(), {0x00, 0xFF, 0x2F, 0x00});
  const size_t total = 14 + 8 + trk.size();
  *size = total;
  if (capacity < total) return 0;
  static const uint8_t head[14] = {'M', 'T', 'h', 'd', 0, 0, 0, 6, 0, 1, 0, 1, 480 >> 8, 480 & 0xFF};
  memcpy(buf, head, 14);
  const uint32_t L = static_cast<uint32_t>(trk.size());
  const uint8_t mtrk[8] = {'M', 'T', 'r', 'k', static_cast<uint8_t>(L >> 24), static_cast<uint8_t>(L >> 16),
                           static_cast<uint8_t>(L >> 8), static_cast<uint8_t>(L)};
  memcpy(buf + 14, mtrk, 8);
  memcpy(buf + 22, trk.data(), trk.size());
  return 0;
}

extern "C" int some_notes_midi(const some_notes* n, int sample_rate, double timestep, double tempo, uint8_t* buf, size_t capacity,
                               size_t* size) {
  SOME_REQUIRE(n != nullptr && sample_rate > 0, "some_notes_midi: bad arguments");
  const int clips = some_notes_clips(n);
  if (clips < 0) return -1;
  std::vector<double> offsets(clips);
  std::vector<int32_t> counts(clips);
  std::vector<float> midi;
  std::vector<int32_t> dur;
  std::vector<uint8_t> rest;
  for (int c = 0; c < clips; ++c) {
    int k = 0;
    const float* m;
    const int32_t* d;
    const uint8_t* r;
    int64_t begin;
    if (some_notes_get(n, c, &k, &m, &d, &r, &begin, nullptr)) return -1;
    offsets[c] = static_cast<double>(begin) / sample_rate;
    counts[c] = k;
    midi.insert(midi.end(), m, m + k), dur.insert(dur.end(), d, d + k), rest.insert(rest.end(), r, r + k);
  }
  return some_midi_write(clips, offsets.data(), counts.data(), midi.data(), dur.data(), rest.data(), timestep, tempo, buf, capacity,
                         size);
}
