/* some_transcribe: transcribe a WAV file with a model file written by `python -m some_b200.export`, without Python.
 *
 *   some_transcribe MODEL WAV [DEVICES]
 *
 * Reads a mono RIFF/WAVE file (16-bit PCM, scaled x / 32768 as libsndfile hands it to librosa.load, or 32-bit float) at any
 * rate, runs some_session_transcribe_sliced (resampling to the model's rate on the GPU when needed, then the silence slicer of
 * infer.py) and prints one line per note:
 *
 *   <chunk offset in seconds> <note_midi> <duration in seconds> <rest 0/1>
 *
 * with the duration computed as (double)dur * timestep, the float64 product of me_infer.py:95.  DEVICES is a device index (default
 * 0) or a comma-separated list of them: a replica of the model on each, with the same output. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "some_b200.h"

static uint32_t le32(const unsigned char* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
static uint16_t le16(const unsigned char* p) { return (uint16_t)(p[0] | (p[1] << 8)); }

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

/* Returns the samples (malloc'ed) or NULL with a message on stderr. */
static float* read_wav(const char* path, long long* n_out, int* rate_out) {
  FILE* f = fopen(path, "rb");
  if (!f) {
    fprintf(stderr, "%s: cannot open\n", path);
    return NULL;
  }
  fseek(f, 0, SEEK_END);
  long size = ftell(f);
  fseek(f, 0, SEEK_SET);
  unsigned char* buf = size > 0 ? malloc((size_t)size) : NULL;
  if (!buf || fread(buf, 1, (size_t)size, f) != (size_t)size) {
    fprintf(stderr, "%s: read error\n", path);
    fclose(f);
    free(buf);
    return NULL;
  }
  fclose(f);
  float* out = NULL;
  if (size < 12 || memcmp(buf, "RIFF", 4) != 0 || memcmp(buf + 8, "WAVE", 4) != 0) {
    fprintf(stderr, "%s: not a RIFF/WAVE file\n", path);
    goto done;
  }
  int fmt = 0, channels = 0, bits = 0, rate = 0;
  const unsigned char* data = NULL;
  uint32_t data_len = 0;
  for (long off = 12; off + 8 <= size;) {
    const uint32_t len = le32(buf + off + 4);
    const unsigned char* body = buf + off + 8;
    if (len > (uint64_t)(size - off - 8)) {
      fprintf(stderr, "%s: truncated '%.4s' chunk\n", path, (const char*)(buf + off));
      goto done;
    }
    if (memcmp(buf + off, "fmt ", 4) == 0 && len >= 16) {
      fmt = le16(body), channels = le16(body + 2), rate = (int)le32(body + 4), bits = le16(body + 14);
    } else if (memcmp(buf + off, "data", 4) == 0) {
      data = body, data_len = len;
    }
    off += 8 + (long)len + (len & 1);
  }
  if (!data || !rate) {
    fprintf(stderr, "%s: no fmt or data chunk\n", path);
    goto done;
  }
  if (channels != 1) {
    fprintf(stderr, "%s: %d channels; this example reads mono files only\n", path, channels);
    goto done;
  }
  if (!((fmt == 1 && bits == 16) || (fmt == 3 && bits == 32))) {
    fprintf(stderr, "%s: format %d with %d bits per sample; this example reads 16-bit PCM or 32-bit float only\n", path, fmt,
            bits);
    goto done;
  }
  const long long n = data_len / (bits / 8);
  out = malloc(sizeof(float) * (size_t)(n > 0 ? n : 1));
  if (!out) goto done;
  for (long long i = 0; i < n; ++i) {
    if (fmt == 1) {
      out[i] = (float)(int16_t)le16(data + 2 * i) / 32768.0f;
    } else {
      uint32_t u = le32(data + 4 * i);
      memcpy(&out[i], &u, 4);
    }
  }
  *n_out = n;
  *rate_out = rate;
done:
  free(buf);
  return out;
}

int main(int argc, char** argv) {
  if (argc < 3) {
    fprintf(stderr, "usage: %s MODEL WAV [DEVICES]\n", argv[0]);
    return 2;
  }
  int devices[64] = {0};
  const int n_devices = argc > 3 ? parse_devices(argv[3], devices) : 1;
  if (n_devices == 0) {
    fprintf(stderr, "some_transcribe: bad device list '%s' (device indices separated by commas)\n", argv[3]);
    return 2;
  }
  long long n = 0;
  int rate = 0;
  float* samples = read_wav(argv[2], &n, &rate);
  if (!samples) return 1;
  some_session* s = NULL;
  some_notes* notes = NULL;
  some_session_info info;
  int rc = 1;
  if (some_session_open_devices(argv[1], devices, n_devices, &s) != 0 || some_session_get_info(s, &info) != 0 ||
      some_notes_create(&notes) != 0 || some_session_transcribe_sliced(s, samples, n, rate, NULL, notes) != 0) {
    fprintf(stderr, "some_transcribe: %s\n", some_last_error());
    goto done;
  }
  const int chunks = some_notes_clips(notes);
  for (int c = 0; c < chunks; ++c) {
    int count = 0;
    const float* midi;
    const int32_t* dur;
    const uint8_t* rest;
    int64_t begin, end;
    some_notes_get(notes, c, &count, &midi, &dur, &rest, &begin, &end);
    const double offset = (double)begin / info.sample_rate;
    for (int k = 0; k < count; ++k)
      printf("%.17g %.9g %.17g %d\n", offset, midi[k], (double)dur[k] * info.timestep, rest[k] ? 1 : 0);
  }
  rc = 0;
done:
  some_notes_destroy(notes);
  some_session_close(s);
  free(samples);
  return rc;
}
