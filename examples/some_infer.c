/* some_infer: infer.py in C.  Transcribes a WAV, FLAC or AIFF file with a model file written by `python -m some_b200.export` and
 * saves the notes as a MIDI file, without Python.
 *
 *   some_infer MODEL AUDIO [--midi PATH] [--tempo BPM] [--device N[,N...]]
 *
 * The file is decoded on the GPU (librosa.load(AUDIO, sr=None, mono=True)), resampled to the model's rate, cut by the silence
 * slicer of infer.py and transcribed by some_session_transcribe_encoded; the MIDI bytes are those of
 * build_midi_file(offsets, segments, tempo) (some_notes_midi).  The default output is AUDIO with its suffix replaced by .mid
 * (pathlib's with_suffix). */
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

/* pathlib.PurePath(path).with_suffix('.mid'): the suffix of the last component (a leading dot does not start one). */
static char* with_mid_suffix(const char* path) {
  size_t n = strlen(path);
  while (n > 1 && path[n - 1] == '/') --n;                  /* pathlib drops trailing slashes */
  const char* slash = NULL;
  for (size_t i = 0; i < n; ++i)
    if (path[i] == '/') slash = path + i;
  const char* name = slash ? slash + 1 : path;
  const size_t name_len = (size_t)(path + n - name);
  size_t stem = name_len;
  for (size_t i = name_len; i > 1; --i)
    if (name[i - 1] == '.') {
      if (i < name_len) stem = i - 1;                         /* a trailing dot is no suffix */
      break;
    }
  const size_t keep = (size_t)(name - path) + stem;
  char* out = malloc(keep + 5);
  if (!out) return NULL;
  memcpy(out, path, keep);
  memcpy(out + keep, ".mid", 5);
  return out;
}

static unsigned char* read_file(const char* path, long long* size) {
  FILE* f = fopen(path, "rb");
  if (!f) {
    fprintf(stderr, "%s: cannot open\n", path);
    return NULL;
  }
  unsigned char* buf = NULL;
  size_t cap = 0, len = 0, got;
  do {
    if (len == cap) {
      cap = cap ? 2 * cap : (1u << 20);
      unsigned char* b = realloc(buf, cap);
      if (!b) {
        free(buf);
        fclose(f);
        fprintf(stderr, "%s: out of memory\n", path);
        return NULL;
      }
      buf = b;
    }
    got = fread(buf + len, 1, cap - len, f);
    len += got;
  } while (got > 0);
  const int bad = ferror(f);
  fclose(f);
  if (bad) {
    fprintf(stderr, "%s: read error\n", path);
    free(buf);
    return NULL;
  }
  *size = (long long)len;
  return buf;
}

int main(int argc, char** argv) {
  const char* model = NULL;
  const char* audio = NULL;
  const char* midi = NULL;
  double tempo = 120.0;
  int devices[64] = {0}, n_devices = 1, positional = 0;
  for (int i = 1; i < argc; ++i) {
    if (!strcmp(argv[i], "--midi") && i + 1 < argc) midi = argv[++i];
    else if (!strcmp(argv[i], "--tempo") && i + 1 < argc) tempo = atof(argv[++i]);
    else if (!strcmp(argv[i], "--device") && i + 1 < argc) n_devices = parse_devices(argv[++i], devices);
    else if (positional == 0) model = argv[i], ++positional;
    else if (positional == 1) audio = argv[i], ++positional;
    else positional = 3;
  }
  if (!model || !audio || positional != 2 || n_devices == 0) {
    fprintf(stderr, "usage: %s MODEL AUDIO [--midi PATH] [--tempo BPM] [--device N[,N...]]\n", argv[0]);
    return 2;
  }
  long long n_bytes = 0;
  unsigned char* bytes = read_file(audio, &n_bytes);
  if (!bytes) return 1;
  char* out_path = midi ? NULL : with_mid_suffix(audio);
  const char* path = midi ? midi : out_path;
  some_session* s = NULL;
  some_notes* notes = NULL;
  some_session_info info;
  uint8_t* buf = NULL;
  int rc = 1;
  const some_encoded item = {bytes, n_bytes};
  size_t size = 0;
  if (!path || some_session_open_devices(model, devices, n_devices, &s) != 0 || some_session_get_info(s, &info) != 0 ||
      some_notes_create(&notes) != 0 || some_session_transcribe_encoded(s, &item, 1, NULL, &notes) != 0 ||
      some_notes_midi(notes, info.sample_rate, info.timestep, tempo, NULL, 0, &size) != 0 || !(buf = malloc(size)) ||
      some_notes_midi(notes, info.sample_rate, info.timestep, tempo, buf, size, &size) != 0) {
    fprintf(stderr, "some_infer: %s\n", path ? some_last_error() : "out of memory");
    goto done;
  }
  FILE* f = fopen(path, "wb");
  const int written = f && fwrite(buf, 1, size, f) == size;
  if (!f || fclose(f) != 0 || !written) {
    fprintf(stderr, "some_infer: cannot write %s\n", path);
    goto done;
  }
  printf("MIDI file saved at: '%s'\n", path);
  rc = 0;
done:
  free(buf);
  some_notes_destroy(notes);
  some_session_close(s);
  free(out_path);
  free(bytes);
  return rc;
}
