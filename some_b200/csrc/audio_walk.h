// The container walk of some_audio_info and the FLAC frame chain of some_flac_chain, both resumable: an encoded stream feeds
// them its bytes as they arrive, and the whole-file functions are the case where everything arrives at once.  Host only.
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/some_b200.h"

namespace some {

// RIFF/WAVE, AIFF / AIFF-C or FLAC metadata, fed in pieces.  Each feed costs time in proportion to its own bytes: the walker holds only the
// bytes of the structure it is reading (at most 48), never those of skipped chunks, tags or metadata blocks, and never the
// audio.  AIFF is read the same way in both modes: COMM must come before SSND, and the walk ends with the SSND chunk.  The rules that depend on where the file ends (a data chunk cut short, "Unexpected end of file", ...) apply when
// the end is signalled, so a refusal comes with some_audio_info's message and offset as soon as it is certain.
//   stream: a second WAV data chunk, or a fmt chunk after the data chunk, is refused when its header is reached (a stream
// cannot take back the samples of the first data chunk, nor change the format they were decoded in); otherwise the last data
// chunk and the last fmt chunk count, as scipy reads them.
class AudioWalk {
 public:
  explicit AudioWalk(bool stream) : stream_(stream) {}
  // Feeds the next n bytes (end: they are the file's last).  Returns -1 with the refusal, else 0 and *known (whether meta()
  // holds the stream's metadata: WAV / AIFF once the data / SSND chunk's header is read, FLAC after the last metadata block;
  // final after the end).  The audio bytes of this feed are the file offsets [*audio_begin, *audio_end) (empty when equal):
  // WAV / AIFF sample bytes within the data / SSND chunk's stated size, FLAC everything after the metadata.  The first held_audio().size() of them
  // are in held_audio() (bytes a header rule had looked ahead at), until the next feed; the rest are in `data`.
  int feed(const uint8_t* data, long long n, bool end, int* known, long long* audio_begin, long long* audio_end);
  const some_audio_meta& meta() const { return m_; }
  const std::vector<uint8_t>& held_audio() const { return held_audio_; }
  long long received() const { return received_; }
  // The bytes the walker holds: at most 48 (the longest header rule's lookahead), of which held_header() are still to be
  // walked and the rest are held_audio().
  long long held() const { return static_cast<long long>(buf_.size() + held_audio_.size()); }
  long long held_header() const { return static_cast<long long>(buf_.size()); }

 private:
  enum Phase { kStart, kMagic, kFlacBlock, kFlacEnd, kFlacAudio, kWavChunk, kAiffChunk, kPcmData, kDone };   // kPcmData: a WAV data or AIFF SSND chunk
  enum { kAdvanced = 0, kMore = 1, kFailed = -1 };
  int step(bool at_end, long long n);
  int data_done(long long avail);
  int wav_done();
  int aiff_chunk(bool at_end, long long p, long long avail, const uint8_t* q);

  const bool stream_;
  Phase phase_ = kStart;
  bool known_ = false, failed_ = false;
  long long received_ = 0, pos_ = 0, need_ = 0, bpos_ = 0;
  std::vector<uint8_t> buf_, held_audio_;   // buf_: the bytes [bpos_, bpos_ + size) that have arrived
  uint8_t head_[12] = {};                   // the file's first bytes (audio.decode_wav names the container by them)
  long long head_len_ = 0;
  some_audio_meta m_{};
  // FLAC: the first metadata block is STREAMINFO; a skipped block's header offset, until its end arrives
  bool first_ = true;
  long long flac_off_ = 0, skipped_ = -1;
  int min_bs_ = 0, max_bs_ = 0, rate_ = 0, channels_ = 0, bps_ = 0;
  long long length_ = 0;
  // WAV: scipy's walk; the end of the last fmt chunk, until it has arrived (scipy stops at the end of the file)
  long long file_size_ = 0, fmt_end_ = -1;
  int fmt_pad_ = 0;
  bool have_fmt_ = false, have_data_ = false;
  int tag_ = 0, block_align_ = 0, bits_ = 0;
  int d_kind_ = 0, d_channels_ = 0, d_bits_ = 0, d_isz_ = 0, d_bps_ = 0;
  long long d_size_ = 0, d_begin_ = 0, d_end_ = 0, d_frames_ = 0, d_offset_ = 0, d_bytes_ = 0;
  // AIFF: the end of the FORM chunk (it bounds the walk), whether the form type is AIFC and COMM has been read (its format
  // is in channels_, rate_, bits_ and d_kind_ / d_isz_)
  long long form_end_ = 0;
  bool aifc_ = false, have_comm_ = false;
};

// One recording's frame chain, resumable: where the next frame must start (a file offset), the samples and frames chained so
// far and the blocking strategy (-1 before the first frame).
struct FlacWalk {
  long long pos = 0, got = 0, count = 0;
  int strategy = -1;
  bool done = false;
};
// Continues `w` over the candidates frames[*i ..] (in byte order) of a window of the file: file offset x lies at x + base in
// the candidates' coordinates and the window's bytes end at `stop` there.  Appends the chained candidate indices to
// chain[*k .. capacity).  final: the window runs to the end of the file, and every check of some_flac_chain applies with its
// message; before that, the walk waits without error at a frame that is SOME_FLAC_TRUNCATED (its window ends) or where fewer
// than 16 bytes (the longest frame header) are left and no header was found.  Returns -1 with the refusal, else 0.
int flac_walk(const some_flac_frame* frames, int n_frames, int* i, long long base, long long stop, long long total, bool final,
              FlacWalk* w, int32_t* chain, int capacity, int* k);

}  // namespace some
