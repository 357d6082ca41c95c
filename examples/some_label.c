/* some_label: batch_infer.py in C.  Labels a DiffSinger dataset with a model file written by `python -m some_b200.export`:
 * writes note_seq / note_dur for every item of DATASET/transcriptions.csv, without Python.
 *
 *   some_label MODEL DATASET [--csv PATH] [--round-midi] [--overwrite] [--device N[,N...]]
 *
 * Item `name` is read from DATASET/wavs/{name}.wav (WAV, FLAC or AIFF bytes), decoded on the GPU, cut by the silence slicer
 * and transcribed by some_session_label_dataset, which writes the same file as batch_infer.py's command with the same notes.
 * The default output is DATASET/transcriptions.csv itself, which needs --overwrite. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "some_b200.h"

/* Parses a device list: one index, or several separated by commas ("0,1").  Returns the count (at most 64), or 0 when the
 * list is malformed. */
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

static void warn_missing(const char* path, void* user) {
  (void)user;
  printf("WARNING: audio file does not exist: '%s'\n", path);
}

int main(int argc, char** argv) {
  const char* model = NULL;
  const char* dataset = NULL;
  const char* csv = NULL;
  int round_midi = 0, overwrite = 0, devices[64] = {0}, n_devices = 1, positional = 0;
  for (int i = 1; i < argc; ++i) {
    if (!strcmp(argv[i], "--csv") && i + 1 < argc) csv = argv[++i];
    else if (!strcmp(argv[i], "--round-midi")) round_midi = 1;
    else if (!strcmp(argv[i], "--overwrite")) overwrite = 1;
    else if (!strcmp(argv[i], "--device") && i + 1 < argc) n_devices = parse_devices(argv[++i], devices);
    else if (positional == 0) model = argv[i], ++positional;
    else if (positional == 1) dataset = argv[i], ++positional;
    else positional = 3;
  }
  if (!model || !dataset || positional != 2 || n_devices == 0) {
    fprintf(stderr, "usage: %s MODEL DATASET [--csv PATH] [--round-midi] [--overwrite] [--device N[,N...]]\n", argv[0]);
    return 2;
  }
  some_session* s = NULL;
  int rc = 1;
  if (some_session_open_devices(model, devices, n_devices, &s) != 0 ||
      some_session_label_dataset(s, dataset, csv, round_midi, overwrite, NULL, warn_missing, NULL, NULL) != 0) {
    fprintf(stderr, "some_label: %s\n", some_last_error());
    goto done;
  }
  rc = 0;
done:
  fflush(stdout);
  some_session_close(s);
  return rc;
}
