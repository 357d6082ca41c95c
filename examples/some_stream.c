/* some_stream: transcribe a recording while it arrives, with a model file written by `python -m some_b200.export`, without
 * Python.
 *
 *   some_stream [--peek MS] [--frames] MODEL RATE [DEVICES] < pcm
 *   some_stream [--peek MS] [--frames] MODEL - [DEVICES] < file.wav, file.flac or file.aif
 *
 * With RATE, reads raw mono little-endian float32 samples at RATE Hz from stdin in blocks of 100 ms and pushes each block to a
 * some_stream.  With `-`, reads a WAV, FLAC or AIFF byte stream from stdin in 64 KB reads and pushes each read to an encoded
 * stream (some_stream_open_encoded: the rate comes from the header; decoded and down-mixed on the GPU as
 * some_session_transcribe_encoded does).  Prints the notes of every chunk as soon as it is delivered, one line per note:
 *
 *   <chunk offset in seconds> <note_midi> <duration in seconds> <rest 0/1>
 *
 * the same lines examples/some_transcribe prints for the whole recording.  With --peek MS, after each push that completes
 * another MS milliseconds of audio (at most one peek per push), it also prints the provisional notes of the part of the
 * recording no chunk has covered yet (some_stream_peek), in the same format with "~ " in front:
 *
 *   ~ <region offset in seconds> <note_midi> <duration in seconds> <rest 0/1>
 *
 * A later peek or the delivered chunk replaces them.  With --frames, each chunk's (and each peeked region's) note lines are
 * followed by one line per frame of it, from its frame curves (some_notes_get_frames), with "~ " in front for a peek:
 *
 *   f <frame time in seconds> <midi> <rest 0/1> <boundary probability> <1-based note index>
 *
 * frame t of a chunk is centred at its first sample + t * hop.  Live from a microphone:
 *
 *   arecord -f FLOAT_LE -c1 -r 44100 | some_stream model.somemodel 44100
 *   arecord -f S16_LE -c2 -r 48000 -t wav | some_stream model.somemodel - */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "some_b200.h"

/* Parses a device list: one index, or several separated by commas ("0,1"; "0,0" runs two replicas on one GPU).  Returns the
 * count (at most 64), or 0 when the list is malformed. */
static int parse_devices(const char* list, int* devices) {
  int n = 0;
  for (const char* p = list;; ++p) {
    char* end;
    const long v = strtol(p, &end, 10);
    if (end == p || *p == '-' || *p == '+' || v > 1000000 || n == 64 || (*end != ',' && *end != '\0')) return 0;
    devices[n++] = (int)v;
    if (*end == '\0') return n;
    p = end;
  }
}

static int print_frames = 0;             /* --frames */

static void print_chunks(const some_notes* notes, const some_session_info* info, const char* prefix) {
  const int chunks = some_notes_clips(notes);
  for (int c = 0; c < chunks; ++c) {
    int count = 0;
    const float* midi;
    const int32_t* dur;
    const uint8_t* rest;
    int64_t begin, end;
    some_notes_get(notes, c, &count, &midi, &dur, &rest, &begin, &end);
    const double offset = (double)begin / info->sample_rate;
    for (int k = 0; k < count; ++k)
      printf("%s%.17g %.9g %.17g %d\n", prefix, offset, midi[k], (double)dur[k] * info->timestep, rest[k] ? 1 : 0);
    if (!print_frames) continue;
    int frames = 0;
    const float *fm, *fb;
    const uint8_t* fr;
    const int32_t* fn;
    if (some_notes_get_frames(notes, c, &frames, &fm, &fr, &fb, &fn) != 0) continue;
    for (int t = 0; t < frames; ++t)
      printf("%sf %.17g %.9g %d %.9g %d\n", prefix, (double)(begin + (int64_t)t * info->hop) / info->sample_rate, fm[t],
             fr[t] ? 1 : 0, fb[t], fn[t]);
  }
  fflush(stdout);
}

/* --peek MS: peeks and prints once `received` samples at `rate` reach the next multiple of MS milliseconds (peek_ms 0: never). */
typedef struct {
  int peek_ms;
  long long next_ms;
  some_notes* notes;
} peeker;

static int maybe_peek(peeker* p, some_stream* st, long long received, int rate, const some_session_info* info) {
  if (p->peek_ms <= 0 || rate <= 0 || received * 1000 < p->next_ms * rate) return 0;
  if (some_stream_peek(st, p->notes) != 0) return -1;
  print_chunks(p->notes, info, "~ ");
  p->next_ms = (received * 1000 / rate / p->peek_ms + 1) * p->peek_ms;
  return 0;
}

/* `-`: the bytes of a WAV, FLAC or AIFF file from stdin, 64 KB per push. */
static int run_encoded(some_session* s, const some_session_info* info, peeker* pk) {
  static unsigned char buf[1 << 16];
  some_stream* st = NULL;
  some_notes* notes = NULL;
  int rc = 1;
  if (some_notes_create(&notes) != 0 || some_notes_set_frames(notes, print_frames) != 0 ||
      some_stream_open_encoded(s, NULL, &st) != 0)
    goto fail;
  for (;;) {
    const size_t got = fread(buf, 1, sizeof(buf), stdin);
    if (got == 0) break;
    if (some_stream_push_bytes(st, buf, (long long)got, notes) != 0) goto fail;
    print_chunks(notes, info, "");
    some_stream_info si;
    some_audio_meta m;
    if (some_stream_get_info(st, &si) != 0 || some_stream_get_meta(st, &m, NULL, NULL) != 0 ||
        maybe_peek(pk, st, si.received, m.rate, info) != 0)
      goto fail;
  }
  if (ferror(stdin)) {
    fprintf(stderr, "some_stream: read error\n");
    goto done;
  }
  if (some_stream_finish(st, notes) != 0) goto fail;
  print_chunks(notes, info, "");
  rc = 0;
  goto done;
fail:
  fprintf(stderr, "some_stream: %s\n", some_last_error());
done:
  some_stream_close(st);
  some_notes_destroy(notes);
  return rc;
}

int main(int argc, char** argv) {
  peeker pk = {0, 0, NULL};
  for (;;) {
    if (argc >= 3 && strcmp(argv[1], "--peek") == 0) {
      pk.peek_ms = atoi(argv[2]);
      if (pk.peek_ms <= 0) {
        fprintf(stderr, "some_stream: --peek takes a positive number of milliseconds, not '%s'\n", argv[2]);
        return 2;
      }
      pk.next_ms = pk.peek_ms;
      argv[2] = argv[0];
      argc -= 2, argv += 2;
    } else if (argc >= 2 && strcmp(argv[1], "--frames") == 0) {
      print_frames = 1;
      argv[1] = argv[0];
      argc -= 1, argv += 1;
    } else {
      break;
    }
  }
  const int encoded = argc >= 3 && strcmp(argv[2], "-") == 0;
  if (argc < 3 || (!encoded && atoi(argv[2]) <= 0)) {
    fprintf(stderr, "usage: %s [--peek MS] [--frames] MODEL RATE [DEVICES] < mono float32 little-endian PCM\n"
                    "       %s [--peek MS] [--frames] MODEL - [DEVICES] < WAV, FLAC or AIFF bytes\n", argv[0], argv[0]);
    return 2;
  }
  int devices[64] = {0};
  const int n_devices = argc > 3 ? parse_devices(argv[3], devices) : 1;
  if (n_devices == 0) {
    fprintf(stderr, "some_stream: bad device list '%s' (device indices separated by commas)\n", argv[3]);
    return 2;
  }
  if (encoded) {
    some_session* s = NULL;
    some_session_info info;
    int rc = 1;
    if (some_session_open_devices(argv[1], devices, n_devices, &s) != 0 || some_session_get_info(s, &info) != 0 ||
        (pk.peek_ms && (some_notes_create(&pk.notes) != 0 || some_notes_set_frames(pk.notes, print_frames) != 0)))
      fprintf(stderr, "some_stream: %s\n", some_last_error());
    else
      rc = run_encoded(s, &info, &pk);
    some_notes_destroy(pk.notes);
    some_session_close(s);
    return rc;
  }
  const int rate = atoi(argv[2]);
  const size_t block = (size_t)(rate / 10 > 0 ? rate / 10 : 1);
  unsigned char* raw = malloc(4 * block);
  float* samples = malloc(sizeof(float) * block);
  some_session* s = NULL;
  some_stream* st = NULL;
  some_notes* notes = NULL;
  some_session_info info;
  int rc = 1;
  if (!raw || !samples) goto done;
  if (some_session_open_devices(argv[1], devices, n_devices, &s) != 0 || some_session_get_info(s, &info) != 0 ||
      some_notes_create(&notes) != 0 || some_notes_set_frames(notes, print_frames) != 0 ||
      some_stream_open(s, rate, NULL, &st) != 0 ||
      (pk.peek_ms && (some_notes_create(&pk.notes) != 0 || some_notes_set_frames(pk.notes, print_frames) != 0))) {
    fprintf(stderr, "some_stream: %s\n", some_last_error());
    goto done;
  }
  size_t have = 0;                       /* bytes of the current block read so far */
  long long pushed = 0;
  for (;;) {
    const size_t got = fread(raw + have, 1, 4 * block - have, stdin);
    have += got;
    const int eof = got == 0;
    if (have == 4 * block || (eof && have >= 4)) {
      const size_t n = have / 4;
      for (size_t i = 0; i < n; ++i) {
        const unsigned char* p = raw + 4 * i;
        const uint32_t u = p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24);
        memcpy(&samples[i], &u, 4);
      }
      memmove(raw, raw + 4 * n, have - 4 * n);
      have -= 4 * n;
      if (some_stream_push(st, samples, (long long)n, notes) != 0) {
        fprintf(stderr, "some_stream: %s\n", some_last_error());
        goto done;
      }
      print_chunks(notes, &info, "");
      pushed += (long long)n;
      if (maybe_peek(&pk, st, pushed, rate, &info) != 0) {
        fprintf(stderr, "some_stream: %s\n", some_last_error());
        goto done;
      }
    }
    if (eof) break;
  }
  if (ferror(stdin)) {
    fprintf(stderr, "some_stream: read error\n");
    goto done;
  }
  if (some_stream_finish(st, notes) != 0) {
    fprintf(stderr, "some_stream: %s\n", some_last_error());
    goto done;
  }
  print_chunks(notes, &info, "");
  rc = 0;
done:
  some_stream_close(st);
  some_notes_destroy(notes);
  some_notes_destroy(pk.notes);
  some_session_close(s);
  free(raw);
  free(samples);
  return rc;
}
