// Host-only helpers of the encoded-file path (no CUDA call): container metadata (some_audio_info), the FLAC frame chain
// (some_flac_chain) and Standard MIDI File bytes (some_midi_write, some_notes_midi).
//
// some_audio_info reads what some_b200.audio.load accepts (load reads FLAC and AIFF headers through it), except integer
// PCM in 5-8 byte containers (scipy: int64, x / 2^63) and 1-8 bit PCM in wider containers, which it refuses: RIFF/WAVE
// exactly as scipy.io.wavfile.read walks it (the chunk loop bounded by the RIFF size, the pad byte of odd chunks, a data
// chunk cut short by the end of the file), FLAC (oracle/flac.py restates its metadata rules), and AIFF / AIFF-C as
// libsndfile reads them (oracle/aiff.py restates the walk in numpy).  Its refusals carry a reason and a byte offset.
// some_flac_chain is the one copy of the walk FlacBatch used to do in Python; both the Python and the session's paths call it.
// some_midi_write is some_b200.midi.build_midi_file(...).to_bytes(), tick for tick.
#include <limits.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "audio_walk.h"
#include "host_common.h"

#include "../../include/some_b200.h"

using namespace some;

namespace {

uint32_t le32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | (static_cast<uint32_t>(p[3]) << 24); }
uint16_t le16(const uint8_t* p) { return static_cast<uint16_t>(p[0] | (p[1] << 8)); }
uint32_t be32(const uint8_t* p) { return (static_cast<uint32_t>(p[0]) << 24) | (p[1] << 16) | (p[2] << 8) | p[3]; }
int16_t be16(const uint8_t* p) { return static_cast<int16_t>((p[0] << 8) | p[1]); }

// A chunk id or compression type for a message: printable ASCII as is, other bytes as \xNN.
std::string fourcc(const uint8_t* p) {
  std::string s;
  char hex[8];
  for (int i = 0; i < 4; ++i) {
    if (p[i] >= 0x20 && p[i] < 0x7F && p[i] != '\\') s += static_cast<char>(p[i]);
    else snprintf(hex, sizeof(hex), "\\x%02x", p[i]), s += hex;
  }
  return s;
}

// The integer part of an 80-bit IEEE extended value (sign, 15-bit exponent, 64-bit mantissa with its explicit integer bit),
// which is how libsndfile's aiff.c turns COMM's sampleRate into an int; -1 when it is not finite, below 1 or at least 2^31.
// *value: the value as a double, for the message.
long long extended_int(const uint8_t* b, double* value) {
  const int sign = b[0] >> 7, e = ((b[0] & 0x7F) << 8 | b[1]) - 16383;
  uint64_t mant = 0;
  for (int i = 2; i < 10; ++i) mant = mant << 8 | b[i];
  if (e == 0x7FFF - 16383) {
    *value = mant << 1 ? NAN : (sign ? -INFINITY : INFINITY);
    return -1;
  }
  *value = (sign ? -1.0 : 1.0) * ldexp(static_cast<double>(mant), e - 63);
  if (sign || e < 0) return -1;                            // negative, or below 1
  uint64_t ip;
  if (e <= 63) {
    ip = mant >> (63 - e);
  } else {                                                 // an unnormalised mantissa may still give a small value
    const int sh = e - 63;
    if (sh >= 31 || mant >= (uint64_t(1) << (31 - sh))) return -1;
    ip = mant << sh;
  }
  return ip >= 1 && ip < (uint64_t(1) << 31) ? static_cast<long long>(ip) : -1;
}

// The length of an ID3v2 tag: 10 + the syncsafe size (+ 10 with a footer), 0 without a tag.
long long id3_size(const uint8_t* d, long long n) {
  if (n < 10 || memcmp(d, "ID3", 3) != 0) return 0;
  const long long size = (d[6] & 0x7F) << 21 | (d[7] & 0x7F) << 14 | (d[8] & 0x7F) << 7 | (d[9] & 0x7F);
  return 10 + size + ((d[5] & 0x10) ? 10 : 0);
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

// ---------------------------------------------------------------------------------------------------- the container walk
// The feed loop: the bytes [received_, e) arrive; r is the first of them not consumed yet.  Outside the audio, the step at
// pos_ runs on the bytes [pos_, r) held in buf_ (bpos_ == pos_ when it runs) and either advances pos_, asks for more bytes
// (need_ from pos_) or refuses.  Bytes below pos_ that were never held are skipped as they arrive.
int AudioWalk::feed(const uint8_t* data, long long n, bool end, int* known, long long* audio_begin, long long* audio_end) {
  SOME_REQUIRE(!failed_, "the walk was refused before");
  held_audio_.clear();
  const long long r0 = received_, e = received_ + n;
  long long r = r0, ab = -1, ae = -1;
  auto align = [&] {                     // buf_ starts at pos_ again
    if (pos_ <= bpos_) return;
    const size_t drop = static_cast<size_t>(std::min<long long>(pos_ - bpos_, static_cast<long long>(buf_.size())));
    buf_.erase(buf_.begin(), buf_.begin() + drop);
    bpos_ = pos_;
  };
  auto fail = [&] {
    failed_ = true;
    return -1;
  };
  for (;;) {
    if (phase_ == kDone) {
      r = e;
      break;
    }
    if (phase_ == kPcmData || phase_ == kFlacAudio) {
      const long long stop = phase_ == kPcmData ? d_end_ : LLONG_MAX, hi = std::min(stop, e);
      if (hi > pos_) {
        if (r > pos_)                    // audio bytes a step had looked ahead at
          held_audio_.insert(held_audio_.end(), buf_.begin(), buf_.begin() + (std::min(r, hi) - pos_));
        if (ab < 0) ab = pos_;
        ae = hi;
        pos_ = hi;
        align();
        r = std::max(r, hi);
      }
      if (phase_ == kFlacAudio) {
        m_.data_bytes = e - m_.data_offset;
        if (end) phase_ = kDone;
        if (!end) break;
        continue;
      }
      if (pos_ < stop && !end) break;
      if (data_done(pos_ < stop ? e - d_begin_ : d_end_ - d_begin_)) return fail();
      align();
      continue;
    }
    if (pos_ > r) r = std::min(pos_, e);   // skipped bytes
    const bool at_end = end && r == e;
    if (pos_ > r && !at_end) break;
    const int st = step(at_end, r);
    if (st == kFailed) return fail();
    if (st == kMore) {
      if (r == e) break;                 // (at the end a step never asks for more)
      const long long take = std::min(e, pos_ + need_) - r;
      buf_.insert(buf_.end(), data + (r - r0), data + (r - r0) + take);
      r += take;
      continue;
    }
    align();
  }
  received_ = e;
  *known = known_ ? 1 : 0;
  *audio_begin = ab < 0 ? 0 : ab;
  *audio_end = ab < 0 ? 0 : ae;
  return 0;
}

// One structure at p = pos_: `n` is the end of the bytes that have arrived; q holds the bytes [p, n) (none when p > n, at the
// end only).  Before the end, a rule that would read bytes past p + k or depend on where the file ends waits for k bytes.
int AudioWalk::step(bool at_end, long long n) {
  const long long p = pos_, avail = n - p;
  const uint8_t* q = buf_.data();
#define SOME_WAIT(k)                \
  if (!at_end && avail < (k)) {     \
    need_ = (k);                    \
    return kMore;                   \
  }
  switch (phase_) {
    case kStart: {
      SOME_WAIT(12);
      head_len_ = std::min<long long>(avail, 12);
      memcpy(head_, q, static_cast<size_t>(head_len_));
      pos_ = id3_size(q, avail);
      phase_ = kMagic;
      return kAdvanced;
    }
    case kMagic: {
      SOME_WAIT(4);
      if (avail >= 4 && memcmp(q, "fLaC", 4) == 0) {
        flac_off_ = p;
        pos_ = p + 4;
        phase_ = kFlacBlock;
        return kAdvanced;
      }
      if (head_len_ >= 4 && memcmp(head_, "FORM", 4) == 0) {
        SOME_REQUIRE(head_len_ >= 12, "AIFF/IFF: FORM header truncated at byte offset 0");
        aifc_ = memcmp(head_ + 8, "AIFC", 4) == 0;
        SOME_REQUIRE(aifc_ || memcmp(head_ + 8, "AIFF", 4) == 0, "AIFF/IFF: form type '%s' is neither AIFF nor AIFC (at byte "
                     "offset 8); AIFF and AIFF-C files are read", fourcc(head_ + 8).c_str());
        form_end_ = static_cast<long long>(be32(head_ + 4)) + 8;
        pos_ = 12;
        phase_ = kAiffChunk;
        return kAdvanced;
      }
      // p > 0: an ID3v2 tag came first, which only a FLAC stream may have; say where its fLaC marker was looked for
      SOME_REQUIRE(head_len_ >= 12 && memcmp(head_, "RIFF", 4) == 0 && memcmp(head_ + 8, "WAVE", 4) == 0,
                   "not a RIFF/WAVE file (%s%s); some_b200.audio reads WAV files only", not_wave_kind(head_, head_len_).c_str(),
                   p > 0 ? ("; no fLaC marker at byte offset " + std::to_string(p)).c_str() : "");
      file_size_ = static_cast<long long>(le32(head_ + 4)) + 8;
      pos_ = 12;
      phase_ = kWavChunk;
      return kAdvanced;
    }
    // FLAC metadata blocks (audio.parse_flac reads FLAC headers through this walk)
    case kFlacBlock:
    case kFlacEnd: {
      if (skipped_ >= 0) {                 // the skipped block ends at p
        SOME_REQUIRE(n >= p, "FLAC metadata block truncated at byte offset %lld", skipped_);
        skipped_ = -1;
      }
      if (phase_ == kFlacEnd) {
        SOME_REQUIRE(bps_ <= 24,
                     "FLAC stream of %d bits per sample (at byte offset %lld); only up to 24 bits are decoded (libsndfile's "
                     "float scaling is exact up to 24 bits)",
                     bps_, flac_off_ + 8);
        SOME_REQUIRE(rate_ != 0 && max_bs_ != 0, "invalid FLAC STREAMINFO (sample rate %d, max block size %d) at byte offset %lld",
                     rate_, max_bs_, flac_off_ + 8);
        m_.container = SOME_AUDIO_FLAC;
        m_.rate = rate_, m_.channels = channels_, m_.bits = bps_, m_.kind = 0;
        m_.min_blocksize = min_bs_, m_.max_blocksize = max_bs_;
        m_.frames = length_;
        m_.data_offset = p;
        m_.data_bytes = 0;
        known_ = true;
        phase_ = kFlacAudio;
        return kAdvanced;
      }
      SOME_WAIT(4);
      SOME_REQUIRE(avail >= 4, "FLAC metadata block header truncated at byte offset %lld", p);
      const int last = q[0] >> 7, kind = q[0] & 0x7F;
      const long long size = (static_cast<long long>(q[1]) << 16) | (q[2] << 8) | q[3];
      SOME_REQUIRE(!(first_ && (kind != 0 || size != 34)),
                   "FLAC stream does not start with a 34-byte STREAMINFO block (type %d, %lld bytes at byte offset %lld)", kind,
                   size, p);
      SOME_REQUIRE(first_ || (kind != 0 && kind != 127), "%s FLAC metadata block at byte offset %lld",
                   kind == 0 ? "second STREAMINFO" : "invalid", p);
      if (first_) {
        SOME_WAIT(4 + size);
        SOME_REQUIRE(avail >= 4 + size, "FLAC metadata block truncated at byte offset %lld", p);
        const uint8_t* b = q + 4;
        min_bs_ = (b[0] << 8) | b[1];
        max_bs_ = (b[2] << 8) | b[3];
        rate_ = (b[10] << 12) | (b[11] << 4) | (b[12] >> 4);
        channels_ = ((b[12] >> 1) & 7) + 1;
        bps_ = (((b[12] & 1) << 4) | (b[13] >> 4)) + 1;
        length_ = (static_cast<long long>(b[13] & 15) << 32) | (static_cast<long long>(b[14]) << 24) | (b[15] << 16) |
                  (b[16] << 8) | b[17];
        first_ = false;
      } else {
        skipped_ = p;                      // its body is skipped, not held
      }
      pos_ = p + 4 + size;
      if (last) phase_ = kFlacEnd;
      return kAdvanced;
    }
    // scipy.io.wavfile.read's walk over a RIFF/WAVE file (little-endian RIFF only: audio.decode_wav refuses the rest first).
    // pos_ follows the file position scipy's reads and seeks leave, so the chunk loop ends where scipy's does.
    case kWavChunk: {
      if (fmt_end_ >= 0) {                 // a fmt chunk cut short by the end of the file: scipy's position is the end
        if (at_end && n < fmt_end_) pos_ = n + fmt_pad_;
        fmt_end_ = -1;
        if (pos_ != p) return kAdvanced;
      }
      if (p >= file_size_) return wav_done();
      SOME_WAIT(8);
      if (avail <= 0) {
        SOME_REQUIRE(have_data_, "RIFF/WAVE: Unexpected end of file. (at byte offset %lld)", p);
        return wav_done();
      }
      if (avail < 4) {
        SOME_REQUIRE(have_fmt_ && have_data_, "RIFF/WAVE: Incomplete chunk ID (at byte offset %lld)", p);
        return wav_done();                 // scipy warns and stops at the end of the file
      }
      const bool is_fmt = memcmp(q, "fmt ", 4) == 0, is_data = memcmp(q, "data", 4) == 0;
      if (!is_fmt && !is_data) {           // fact, LIST, JUNK, Fake and unknown chunks: skipped
        if (avail == 4) {
          pos_ = n;
          return kAdvanced;
        }
        SOME_REQUIRE(avail >= 8, "RIFF/WAVE: '%.4s' chunk size truncated at byte offset %lld", q, p);
        const long long size = le32(q + 4);
        pos_ = p + 8 + size + (size & 1);
        return kAdvanced;
      }
      SOME_REQUIRE(avail >= 8, "RIFF/WAVE: '%.4s' chunk size truncated at byte offset %lld", q, p);
      const long long size = le32(q + 4);
      if (is_fmt) {
        SOME_REQUIRE(!(stream_ && d_begin_), "RIFF/WAVE: a fmt chunk after the data chunk at byte offset %lld; an encoded stream "
                     "takes its format from the fmt chunk before its data (a whole file is read with its last, as scipy reads it)",
                     p);
        SOME_REQUIRE(size >= 16, "RIFF/WAVE: Binary structure of wave file is not compliant (fmt chunk of %lld bytes at byte "
                     "offset %lld)", size, p);
        SOME_WAIT(24);
        SOME_REQUIRE(avail >= 24, "RIFF/WAVE: fmt chunk truncated at byte offset %lld", p);
        const uint8_t* b = q + 8;
        int tag = le16(b);
        channels_ = le16(b + 2), rate_ = static_cast<int>(le32(b + 4)), block_align_ = le16(b + 12), bits_ = le16(b + 14);
        const uint32_t byte_rate = le32(b + 8);
        if (tag == 0xFFFE && size >= 18) {
          SOME_WAIT(26);
          SOME_REQUIRE(avail >= 26, "RIFF/WAVE: fmt chunk truncated at byte offset %lld", p);
          const int ext = le16(b + 16);
          SOME_REQUIRE(ext >= 22, "RIFF/WAVE: Binary structure of wave file is not compliant (extension of %d bytes at byte "
                       "offset %lld)", ext, p);
          static const uint8_t tail[12] = {0x00, 0x00, 0x10, 0x00, 0x80, 0x00, 0x00, 0xAA, 0x00, 0x38, 0x9B, 0x71};
          SOME_WAIT(8 + 18 + 22);
          if (avail >= 8 + 18 + 22 && memcmp(b + 18 + 6 + 4, tail, 12) == 0) tag = static_cast<int>(le32(b + 18 + 6));
        }
        tag_ = tag;
        SOME_REQUIRE(tag == 1 || tag == 3, "RIFF/WAVE: Unknown wave file format: %#06x. Supported formats: PCM, IEEE_FLOAT (fmt "
                     "chunk at byte offset %lld)", tag, p);
        SOME_REQUIRE(tag != 1 || byte_rate == static_cast<uint32_t>(rate_) * static_cast<uint32_t>(block_align_),
                     "RIFF/WAVE: WAV header is invalid: nAvgBytesPerSec must equal product of nSamplesPerSec and nBlockAlign, "
                     "but file has nSamplesPerSec = %d, nBlockAlign = %d, and nAvgBytesPerSec = %u (fmt chunk at byte offset "
                     "%lld)", rate_, block_align_, byte_rate, p);
        fmt_end_ = p + 8 + size, fmt_pad_ = size & 1;
        pos_ = fmt_end_ + fmt_pad_;
        have_fmt_ = true;
        return kAdvanced;
      }
      // data
      SOME_REQUIRE(!(stream_ && d_begin_), "RIFF/WAVE: a second data chunk at byte offset %lld; an encoded stream reads one data "
                   "chunk (a whole file is read to its last, as scipy reads it)", p);
      SOME_REQUIRE(have_fmt_, "RIFF/WAVE: No fmt chunk before data (data chunk at byte offset %lld)", p);
      SOME_REQUIRE(channels_ > 0 && block_align_ / channels_ > 0,
                   "RIFF/WAVE: %d channels in blocks of %d bytes (data chunk at byte offset %lld)", channels_, block_align_, p);
      const int bps = block_align_ / channels_;   // scipy's container size
      int kind = 0, isz = bps;
      if (tag_ == 1) {
        SOME_REQUIRE(bits_ <= 64, "RIFF/WAVE: Unsupported bit depth: the WAV file has %d-bit integer data. (data chunk at byte "
                     "offset %lld)", bits_, p);
        if (bits_ >= 1 && bits_ <= 8) kind = bps == 1 ? SOME_PCM_U8 : 0, isz = 1;
        else kind = bps == 2 ? SOME_PCM_S16 : bps == 3 ? SOME_PCM_S24 : bps == 4 ? SOME_PCM_S32 : 0;
        SOME_REQUIRE(kind, "RIFF/WAVE: %d-bit PCM in %d-byte containers is not read (u8, s16, s24 and s32 are; data chunk at "
                     "byte offset %lld)", bits_, bps, p);
      } else {
        SOME_REQUIRE(bits_ == 32 || bits_ == 64, "RIFF/WAVE: Unsupported bit depth: the WAV file has %d-bit floating-point data. "
                     "(data chunk at byte offset %lld)", bits_, p);
        kind = bps == 4 ? SOME_PCM_F32 : bps == 8 ? SOME_PCM_F64 : 0;
        SOME_REQUIRE(kind, "RIFF/WAVE: %d-bit float in %d-byte containers (data chunk at byte offset %lld)", bits_, bps, p);
      }
      d_kind_ = kind, d_channels_ = channels_, d_bits_ = bits_, d_isz_ = isz, d_bps_ = bps, d_size_ = size;
      d_begin_ = p + 8;
      d_end_ = d_begin_ + (kind == SOME_PCM_S24 ? size : size / bps * isz);   // whole items of the stated size
      m_.container = SOME_AUDIO_WAV;
      m_.rate = rate_, m_.channels = channels_, m_.bits = bits_, m_.kind = kind;
      m_.min_blocksize = 0, m_.max_blocksize = 0;
      m_.frames = (d_end_ - d_begin_) / isz / channels_, m_.data_offset = d_begin_, m_.data_bytes = d_end_ - d_begin_;
      known_ = true;
      pos_ = d_begin_;
      phase_ = kPcmData;
      return kAdvanced;
    }
    case kAiffChunk:
      return aiff_chunk(at_end, p, avail, q);
    default:
      return kAdvanced;
  }
}

// libsndfile's walk over a FORM/AIFF or FORM/AIFC file (aiff.c), as oracle/aiff.py restates it: big-endian chunks padded to
// an even length, within the FORM size; COMM gives the format, SSND the samples, and every other chunk is skipped unread.
// The walk ends at the SSND chunk, so both modes read the same: COMM must come before it, and a later COMM or SSND is never
// seen.  The frames are the whole frames of the SSND bytes within its stated size and the file (COMM's numSampleFrames is
// not used), libsndfile's count for a file cut short or written with placeholder sizes.
int AudioWalk::aiff_chunk(bool at_end, long long p, long long avail, const uint8_t* q) {
  auto walk_end = [&] {
    set_error("AIFF/IFF: no %s chunk before byte offset %lld", have_comm_ ? "SSND" : "COMM", p);
    return kFailed;
  };
  if (p + 8 > form_end_) return walk_end();     // no chunk header left within the FORM size
  SOME_WAIT(8);
  if (avail < 8) return walk_end();              // the file ends
  const long long size = be32(q + 4);
  if (memcmp(q, "COMM", 4) == 0) {
    const int need = aifc_ ? 22 : 18;            // AIFF-C: the compression type; its pascal-string name is not read
    SOME_REQUIRE(size >= need, "AIFF/IFF: COMM chunk of %lld bytes at byte offset %lld (%s needs %d)", size, p,
                 aifc_ ? "AIFF-C" : "AIFF", need);
    SOME_WAIT(8 + need);
    SOME_REQUIRE(avail >= 8 + need, "AIFF/IFF: COMM chunk truncated at byte offset %lld", p);
    const uint8_t* b = q + 8;
    const int channels = be16(b), bits = be16(b + 6);
    SOME_REQUIRE(channels >= 1, "AIFF/IFF: %d channels (COMM chunk at byte offset %lld)", channels, p);
    static const uint8_t none[4] = {'N', 'O', 'N', 'E'};
    const uint8_t* ct = aifc_ ? b + 18 : none;
    auto is = [&](const char* a, const char* b2) { return memcmp(ct, a, 4) == 0 || (b2 && memcmp(ct, b2, 4) == 0); };
    const std::string name = fourcc(ct);
    int kind = 0;
    bool known_type = true;
    if (is("NONE", "twos") || is("sowt", nullptr)) {
      const bool le = is("sowt", nullptr);
      if (bits >= 1 && bits <= 8) kind = SOME_PCM_S8;
      else if (bits >= 9 && bits <= 16) kind = le ? SOME_PCM_S16 : SOME_PCM_S16BE;
      else if (bits >= 17 && bits <= 24) kind = le ? SOME_PCM_S24 : SOME_PCM_S24BE;
      else if (bits >= 25 && bits <= 32) kind = le ? SOME_PCM_S32 : SOME_PCM_S32BE;
    } else if (is("raw ", nullptr)) {
      kind = bits == 8 ? SOME_PCM_U8 : 0;
    } else if (is("fl32", "FL32")) {
      kind = bits == 32 ? SOME_PCM_F32BE : 0;
    } else if (is("fl64", "FL64")) {
      kind = bits == 64 ? SOME_PCM_F64BE : 0;
    } else if (is("ulaw", "ULAW")) {
      kind = SOME_PCM_ULAW;
    } else if (is("alaw", "ALAW")) {
      kind = SOME_PCM_ALAW;
    } else {
      known_type = false;
    }
    SOME_REQUIRE(known_type, "AIFF/IFF: AIFF-C compression type '%s' is not read (COMM chunk at byte offset %lld); NONE, "
                 "twos, sowt, raw , fl32, fl64, ulaw and alaw are", name.c_str(), p);
    SOME_REQUIRE(kind, "AIFF/IFF: sampleSize %d is not read with compression type '%s' (COMM chunk at byte offset %lld)", bits,
                 name.c_str(), p);
    double value;
    const long long rate = extended_int(b + 8, &value);
    SOME_REQUIRE(rate > 0, "AIFF/IFF: sample rate %g is outside [1, 2^31) (COMM chunk at byte offset %lld)", value, p);
    channels_ = channels, bits_ = bits, rate_ = static_cast<int>(rate);
    d_kind_ = kind, d_isz_ = pcm_sample_bytes(kind);
    have_comm_ = true;
    pos_ = p + 8 + size + (size & 1);
    return kAdvanced;
  }
  if (memcmp(q, "SSND", 4) != 0) {               // FVER, MARK, INST, COMT, NAME, ANNO, ID3, APPL, ...: skipped
    pos_ = p + 8 + size + (size & 1);
    return kAdvanced;
  }
  SOME_REQUIRE(have_comm_, "AIFF/IFF: SSND chunk before the COMM chunk at byte offset %lld; the COMM chunk must come first", p);
  SOME_WAIT(16);
  SOME_REQUIRE(avail >= 16, "AIFF/IFF: SSND chunk header truncated at byte offset %lld", p);
  const long long offset = be32(q + 8);          // the blockSize at q + 12 is not used
  SOME_REQUIRE(size >= 8 && offset <= size - 8, "AIFF/IFF: SSND offset %lld past its chunk of %lld bytes at byte offset %lld",
               offset, size, p);
  const long long frame = static_cast<long long>(channels_) * d_isz_;
  d_begin_ = p + 16 + offset;
  d_end_ = d_begin_ + (size - 8 - offset) / frame * frame;   // the whole frames of the stated size
  m_.container = SOME_AUDIO_AIFF;
  m_.rate = rate_, m_.channels = channels_, m_.bits = bits_, m_.kind = d_kind_;
  m_.min_blocksize = 0, m_.max_blocksize = 0;
  m_.frames = (d_end_ - d_begin_) / frame, m_.data_offset = d_begin_, m_.data_bytes = d_end_ - d_begin_;
  known_ = true;
  pos_ = d_begin_;
  phase_ = kPcmData;
  return kAdvanced;
}
#undef SOME_WAIT

// The data (SSND) chunk ends: all its stated bytes arrived, or the file ended `avail` bytes into it (AIFF: avail < 0 when the
// SSND offset points past the end).  AIFF keeps the whole frames and reads nothing after them.
int AudioWalk::data_done(long long avail) {
  if (m_.container == SOME_AUDIO_AIFF) {
    const long long frame = static_cast<long long>(channels_) * d_isz_;
    m_.frames = std::min(d_end_ - d_begin_, std::max(avail, 0ll)) / frame;
    m_.data_bytes = m_.frames * frame;
    phase_ = kDone;
    return 0;
  }
  const long long p = d_begin_ - 8;
  long long samples, consumed;
  if (d_kind_ == SOME_PCM_S24) {         // read as raw bytes, then regrouped by three
    consumed = std::min(d_size_, avail);
    SOME_REQUIRE(consumed % 3 == 0, "RIFF/WAVE: %lld bytes of 24-bit samples are not a whole number of samples (data chunk at "
                 "byte offset %lld)", consumed, p);
    samples = consumed / 3;
  } else {
    const long long want = d_size_ / d_bps_;            // items of isz bytes (u8: one byte each)
    samples = std::min(want, avail / d_isz_);
    consumed = std::min(want * d_isz_, avail);
  }
  SOME_REQUIRE(d_channels_ == 1 || samples % d_channels_ == 0,
               "RIFF/WAVE: %lld samples do not fill whole frames of %d channels (data chunk at byte offset %lld)", samples,
               d_channels_, p);
  have_data_ = true;
  d_frames_ = samples / d_channels_, d_offset_ = d_begin_, d_bytes_ = samples * d_isz_;
  m_.frames = d_frames_, m_.data_bytes = d_bytes_;
  pos_ = d_begin_ + consumed + (d_size_ & 1);
  phase_ = kWavChunk;
  return 0;
}

// The chunk loop ends.
int AudioWalk::wav_done() {
  SOME_REQUIRE(have_fmt_, "RIFF/WAVE: no fmt chunk");
  SOME_REQUIRE(have_data_, "RIFF/WAVE: no data chunk");
  m_.container = SOME_AUDIO_WAV;
  m_.rate = rate_, m_.channels = d_channels_, m_.bits = d_bits_, m_.kind = d_kind_;
  m_.min_blocksize = 0, m_.max_blocksize = 0;
  m_.frames = d_frames_, m_.data_offset = d_offset_, m_.data_bytes = d_bytes_;
  known_ = true;
  phase_ = kDone;
  return kAdvanced;
}

extern "C" int some_audio_info(const void* data, long long n_bytes, some_audio_meta* out) {
  SOME_REQUIRE(out != nullptr && n_bytes >= 0 && (data != nullptr || n_bytes == 0), "some_audio_info: bad arguments");
  AudioWalk w(false);
  int known;
  long long a, b;
  if (w.feed(static_cast<const uint8_t*>(data), n_bytes, true, &known, &a, &b)) return -1;
  *out = w.meta();
  return 0;
}

struct some_audio_walk {
  AudioWalk w;
  explicit some_audio_walk(bool stream) : w(stream) {}
};
extern "C" int some_audio_walk_create(int stream, some_audio_walk** out) {
  SOME_REQUIRE(out != nullptr, "some_audio_walk_create: null pointer");
  *out = new some_audio_walk(stream != 0);
  return 0;
}
extern "C" int some_audio_walk_feed(some_audio_walk* w, const void* data, long long n_bytes, int end, int* known,
                                    some_audio_meta* meta, long long* audio_begin, long long* audio_end, long long* held) {
  SOME_REQUIRE(w != nullptr && known && meta && audio_begin && audio_end && n_bytes >= 0 && (data != nullptr || n_bytes == 0),
               "some_audio_walk_feed: bad arguments");
  if (w->w.feed(static_cast<const uint8_t*>(data), n_bytes, end != 0, known, audio_begin, audio_end)) return -1;
  *meta = w->w.meta();
  if (held) *held = w->w.held();
  return 0;
}
extern "C" int some_audio_walk_destroy(some_audio_walk* w) {
  delete w;
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
  for (int r = 0; r < n_recs; ++r) {
    FlacWalk w;
    w.pos = recs[r].audio_start - recs[r].base;
    if (flac_walk(frames, n_frames, &i, recs[r].base, recs[r].end, recs[r].length, true, &w, chain, capacity, &k)) {
      if (failed) *failed = r;
      return -1;
    }
    first[r + 1] = k;
    lengths[r] = w.got;
  }
  return 0;
}

int some::flac_walk(const some_flac_frame* frames, int n_frames, int* i, long long base, long long stop, long long total,
                    bool final, FlacWalk* w, int32_t* chain, int capacity, int* k) {
  char buf[16];
  long long p = base + w->pos;
  for (;;) {
    if ((total && w->got == total) || (!total && p == stop && final)) {
      w->done = true;
      break;
    }
    if (p >= stop) {
      if (!final) break;
      SOME_REQUIRE(false, "FLAC stream ends at byte offset %lld after %lld of %lld samples", p - base, w->got, total);
    }
    while (*i < n_frames && frames[*i].pos < p) ++*i;
    if (*i >= n_frames || frames[*i].pos != p) {
      if (!final && stop - p < 16) break;        // the header may not have arrived yet
      SOME_REQUIRE(false, "no valid FLAC frame header (sync, reserved code, CRC-8 or STREAMINFO mismatch) at byte offset %lld",
                   p - base);
    }
    const some_flac_frame& f = frames[*i];
    if (f.status) {
      if (!final && f.status == SOME_FLAC_TRUNCATED) break;   // its window ends inside it
      SOME_REQUIRE(false, "FLAC frame at byte offset %lld: %s (at byte offset %lld)", p - base,
                   flac_reason(f.status, buf, sizeof(buf)), static_cast<long long>(f.end) - base);
    }
    if (w->strategy < 0) w->strategy = f.variable;
    const long long want = f.variable ? w->got : w->count;
    SOME_REQUIRE(f.variable == w->strategy && f.number == want,
                 "FLAC frame at byte offset %lld: %s number %lld, expected %lld (gap, overlap or changed blocking strategy)",
                 p - base, f.variable ? "sample" : "frame", static_cast<long long>(f.number), want);
    SOME_REQUIRE(!total || w->got + f.blocksize <= total,
                 "FLAC frame at byte offset %lld decodes past the %lld samples STREAMINFO states", p - base, total);
    SOME_REQUIRE(*k < capacity, "some_flac_chain: more than %d chained frames", capacity);
    w->got += f.blocksize;
    chain[(*k)++] = *i;
    ++w->count;
    p = f.end;
    w->pos = p - base;
  }
  return 0;
}

extern "C" int some_flac_chain_resume(const some_flac_frame* frames, int n_frames, int64_t base, int64_t stop, int64_t length,
                                      int final, some_flac_walk* walk, int32_t* chain, int capacity, int* n_chained) {
  SOME_REQUIRE((frames || n_frames == 0) && walk && n_chained && (chain || capacity == 0) && n_frames >= 0 && capacity >= 0,
               "some_flac_chain_resume: bad arguments");
  FlacWalk w;
  w.pos = walk->pos, w.got = walk->got, w.count = walk->count, w.strategy = walk->strategy, w.done = walk->done != 0;
  int i = 0;
  *n_chained = 0;
  const int rc = w.done ? 0 : flac_walk(frames, n_frames, &i, base, stop, length, final != 0, &w, chain, capacity, n_chained);
  walk->pos = w.pos, walk->got = w.got, walk->count = w.count, walk->strategy = w.strategy, walk->done = w.done;
  return rc;
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
