// Host-only (no CUDA call of its own): batch_infer.py's labelling of a DiffSinger dataset, from notes to transcriptions.csv.
//
// some_label_write restates some_b200/batch.py (the specification, pinned to the unmodified reference by
// tests/golden/host_rows.npz): calc_seq, note_timeline, word_durations, align_to_words, notes_touching, dominant_note and
// row_notes, with Python's arithmetic where it decides a digit:
//   - round(x, n) is correctly rounded on the binary value (CPython's dtoa): fixed-point digits of the exact value, then
//     parsed back; x * 1e6 and rint would round some 7th-decimal ties the other way;
//   - str(float) is the shortest repr that reads back, in exponent form below 1e-4 and from 1e16 on (5e-05, 1e+16);
//   - sum() over floats is Neumaier-compensated (CPython 3.12); an int start (0) is added to the first float as an int;
//   - the word clock starts as the int 0, so leading words without phonemes are ints and print as "0".
// some_session_label_dataset is the command of batch_infer.py:149-226 as batch.batch_infer_dataset runs it with
// load_audio=audio.load_native: the csv module's excel dialect on both sides, the notes from
// some_session_transcribe_encoded, groups of rows under a frame budget read on a worker thread.
#include <errno.h>
#include <locale.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>

#include <charconv>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "host_common.h"

#include "../../include/some_b200.h"

using namespace some;

namespace {

// ---------------------------------------------------------------------------------------------- Python's numbers
// A Python number as the labelling meets it: a float, or an int.  The only ints are the word clock before its first
// phoneme and what is computed from it alone (always 0); they print without ".0".
struct Num {
  double v;
  bool is_int;
};
Num flt(double v) { return {v, false}; }
Num add(Num a, Num b) { return {a.v + b.v, a.is_int && b.is_int}; }
Num sub(Num a, Num b) { return {a.v - b.v, a.is_int && b.is_int}; }
Num py_min(Num a, Num b) { return b.v < a.v ? b : a; }     // min(a, b): a unless b < a
Num py_max(Num a, Num b) { return b.v > a.v ? b : a; }     // max(a, b): a unless b > a

locale_t c_locale() {
  static const locale_t loc = newlocale(LC_ALL_MASK, "C", static_cast<locale_t>(0));
  return loc;
}

// round(x, nd) of a float: the exact value's nd-decimal digits, rounded half to even, read back.
double round_digits(double x, int nd) {
  if (!isfinite(x)) return x;
  char buf[400];
  const auto r = std::to_chars(buf, buf + sizeof(buf) - 1, x, std::chars_format::fixed, nd);
  *r.ptr = '\0';
  return strtod_l(buf, nullptr, c_locale());
}
Num round6(Num a) { return a.is_int ? a : flt(round_digits(a.v, 6)); }

// sum(xs) of CPython 3.12: ints added exactly while they lead, the first float added to their total, then Neumaier's
// compensated loop over floats (ints in it are added plainly), the compensation applied at the end when finite and non-zero.
Num py_sum(const std::vector<Num>& xs, size_t a, size_t b) {
  size_t i = a;
  double total = 0;
  for (; i < b && xs[i].is_int; ++i) total += xs[i].v;
  if (i == b) return {total, true};
  double f = total + xs[i++].v, c = 0;
  for (; i < b; ++i) {
    const double x = xs[i].v;
    if (xs[i].is_int) {
      f += x;
      continue;
    }
    const double t = f + x;
    if (fabs(f) >= fabs(x)) c += (f - t) + x;
    else c += (x - t) + f;
    f = t;
  }
  if (c != 0 && isfinite(c)) f += c;
  return flt(f);
}

// str() of a float: CPython's repr (shortest digits that read back; exponent form when the decimal point would sit more
// than 4 places left of the first digit or more than 16 right of it).
std::string py_repr(double x) {
  if (isnan(x)) return "nan";
  if (isinf(x)) return x > 0 ? "inf" : "-inf";
  if (x == 0) return signbit(x) ? "-0.0" : "0.0";
  char buf[64];
  const auto r = std::to_chars(buf, buf + sizeof(buf) - 1, x, std::chars_format::scientific);
  *r.ptr = '\0';
  std::string out = x < 0 ? "-" : "", digits;
  const char* p = buf + (x < 0);
  for (; p < r.ptr && *p != 'e'; ++p)
    if (*p != '.') digits += *p;
  const int exp10 = atoi(p + 1), decpt = exp10 + 1;
  const int nd = static_cast<int>(digits.size());
  if (decpt <= -4 || decpt > 16) {
    out += digits[0];
    if (nd > 1) out += "." + digits.substr(1);
    char e[16];
    snprintf(e, sizeof(e), "e%c%02d", exp10 < 0 ? '-' : '+', abs(exp10));
    out += e;
  } else if (decpt <= 0) {
    out += "0." + std::string(-decpt, '0') + digits;
  } else if (decpt < nd) {
    out += digits.substr(0, decpt) + "." + digits.substr(decpt);
  } else {
    out += digits + std::string(decpt - nd, '0') + ".0";
  }
  return out;
}
std::string py_str(Num a) {
  if (!a.is_int) return py_repr(a.v);
  char buf[32];
  snprintf(buf, sizeof(buf), "%lld", static_cast<long long>(a.v));
  return buf;
}

// float(tok) for the forms DiffSinger writes: [+-] digits [. digits] [(e|E) [+-] digits], at least one mantissa digit.
bool parse_float(const std::string& tok, double* out) {
  size_t i = 0, n = tok.size(), mant = 0;
  if (i < n && (tok[i] == '+' || tok[i] == '-')) ++i;
  for (; i < n && tok[i] >= '0' && tok[i] <= '9'; ++i) ++mant;
  if (i < n && tok[i] == '.')
    for (++i; i < n && tok[i] >= '0' && tok[i] <= '9'; ++i) ++mant;
  if (!mant) return false;
  if (i < n && (tok[i] == 'e' || tok[i] == 'E')) {
    ++i;
    if (i < n && (tok[i] == '+' || tok[i] == '-')) ++i;
    size_t ed = 0;
    for (; i < n && tok[i] >= '0' && tok[i] <= '9'; ++i) ++ed;
    if (!ed) return false;
  }
  if (i != n) return false;
  *out = strtod_l(tok.c_str(), nullptr, c_locale());      // correctly rounded, like float(); overflow gives inf as float() does
  return true;
}

// int(tok) for [+-] digits (at most 18 of them).
bool parse_int(const std::string& tok, long long* out) {
  size_t i = (!tok.empty() && (tok[0] == '+' || tok[0] == '-')) ? 1 : 0;
  if (i == tok.size() || tok.size() - i > 18) return false;
  long long v = 0;
  for (size_t k = i; k < tok.size(); ++k) {
    if (tok[k] < '0' || tok[k] > '9') return false;
    v = v * 10 + (tok[k] - '0');
  }
  *out = tok[0] == '-' ? -v : v;
  return true;
}

std::vector<std::string> split_spaces(const char* s) {      // str.split(' '): every single space separates
  std::vector<std::string> out(1);
  for (; *s; ++s) {
    if (*s == ' ') out.emplace_back();
    else out.back() += *s;
  }
  return out;
}

// ---------------------------------------------------------------------------------------------- batch.py, restated
const char* const kNoteNames[12] = {"C", "C#", "D", "D#", "E", "F", "F#", "G", "G#", "A", "A#", "B"};

// calc_seq: note name (sharps, octave int(num / 12) - 1) and the signed cents int(round(m - round(m, 0), 2) * 100).
int calc_seq(double m, bool rest, std::string* out) {
  if (rest) {
    *out = "rest";
    return 0;
  }
  SOME_REQUIRE(isfinite(m) && fabs(m) < 9007199254740992.0, "note pitch %g is not a finite MIDI value", m);
  const double nearest = rint(m);                            // round(m, 0): half to even
  const long long cent = static_cast<long long>(round_digits(m - nearest, 2) * 100);   // int() truncates: 28.999... -> 28
  const long long num = static_cast<long long>(nearest);
  *out = std::string(kNoteNames[((num % 12) + 12) % 12]) +
         std::to_string(static_cast<long long>(static_cast<double>(num) / 12.0) - 1);
  if (cent > 0) *out += "+" + std::to_string(cent);
  else if (cent < 0) *out += std::to_string(cent);
  return 0;
}

struct Note {
  Num start, end, dur;
  std::string seq;
};

// note_timeline: chunk-relative notes -> absolute records rounded to 6 decimals, each start clipped at the previous end.
int note_timeline(int n_chunks, const double* offsets, const int32_t* counts, const float* note_midi, const int32_t* note_dur,
                  const uint8_t* note_rest, double timestep, std::vector<Note>* notes) {
  int64_t a = 0;
  for (int c = 0; c < n_chunks; ++c) {
    SOME_REQUIRE(counts[c] >= 0, "chunk %d has %d notes", c, counts[c]);
    SOME_REQUIRE(counts[c] == 0 || (note_midi && note_dur && note_rest), "null note arrays");
    const Num offset = round6(flt(offsets[c]));
    Num elapsed = {0, true};
    for (int j = 0; j < counts[c]; ++j, ++a) {
      const Num d = round6(flt(static_cast<double>(note_dur[a]) * timestep));
      elapsed = round6(elapsed);
      Note rec;
      rec.start = round6(add(offset, elapsed));
      rec.end = round6(add(add(offset, elapsed), d));
      if (calc_seq(note_midi[a], note_rest[a] != 0, &rec.seq)) return -1;
      if (!notes->empty() && rec.start.v < notes->back().end.v) rec.start = notes->back().end;
      rec.dur = round6(sub(rec.end, rec.start));
      notes->push_back(rec);
      elapsed = add(elapsed, d);
    }
  }
  return 0;
}

// The indices [*lo, *hi) of Python's xs[a:b] over n items.
void py_slice(long long n, long long a, long long b, long long* lo, long long* hi) {
  auto clamp = [n](long long i) { return i < 0 ? std::max(0LL, i + n) : std::min(i, n); };
  *lo = clamp(a), *hi = std::max(clamp(b), *lo);
}

struct Span {
  Num start, end;
};

// row_notes with word_durations, align_to_words, notes_touching and dominant_note: the note_seq / note_dur fields.
int row_fields(std::vector<Note>& notes, const char* ph_dur_field, const char* ph_num_field, bool round_midi, std::string* seq_out,
               std::string* dur_out) {
  SOME_REQUIRE(ph_dur_field && ph_num_field, "ph_dur / ph_num field is NULL");
  std::vector<Num> ph_dur;
  std::vector<long long> ph_num;
  for (const std::string& tok : split_spaces(ph_dur_field)) {
    double v;
    SOME_REQUIRE(parse_float(tok, &v), "ph_dur value %zu '%s' is not a decimal number", ph_dur.size(), tok.c_str());
    ph_dur.push_back(round6(flt(v)));
  }
  for (const std::string& tok : split_spaces(ph_num_field)) {
    long long v;
    SOME_REQUIRE(parse_int(tok, &v), "ph_num value %zu '%s' is not an integer", ph_num.size(), tok.c_str());
    ph_num.push_back(v);
  }
  std::vector<Span> words;                                   // word_durations
  long long first = 0;
  Num t = {0, true};
  for (long long count : ph_num) {
    long long lo, hi;
    py_slice(static_cast<long long>(ph_dur.size()), first, first + count, &lo, &hi);
    const Num length = round6(py_sum(ph_dur, lo, hi));
    words.push_back({round6(t), round6(add(t, length))});
    first += count;
    t = add(t, length);
  }
  std::vector<Num> edges;                                     // align_to_words
  for (const Span& w : words) edges.push_back(w.start);
  edges.push_back(words.back().end);
  const double tol = 0.05;
  std::vector<const Note*> kept;
  for (Note& rec : notes) {
    for (const Num& e : edges) {
      if (e.v - tol <= rec.start.v && rec.start.v <= e.v + tol) rec.start = e;
      if (e.v - tol <= rec.end.v && rec.end.v <= e.v + tol) rec.end = e;
    }
    rec.dur = round6(sub(rec.end, rec.start));
    if (rec.dur.v > 0) kept.push_back(&rec);
  }
  std::vector<const std::string*> seq;
  std::vector<Num> dur;
  for (const Span& w : words) {
    const Num word_len = round6(sub(w.end, w.start));
    if (round_midi) {                                         // dominant_note
      const std::string* best = nullptr;
      Num best_overlap = {0, true};
      for (const Note* n : kept) {
        const Num overlap = py_max({0, true}, sub(py_min(w.end, n->end), py_max(w.start, n->start)));
        if (overlap.v > best_overlap.v) best_overlap = overlap, best = &n->seq;
      }
      static const std::string rest = "rest";
      seq.push_back(best ? best : &rest);
      dur.push_back(word_len);
      continue;
    }
    const size_t s0 = seq.size();
    std::vector<Num> w_dur;
    for (const Note* n : kept) {                              // notes_touching
      const double lo = w.start.v, hi = w.end.v, a = n->start.v, b = n->end.v;
      if (!((lo < a && a < hi) || (lo < b && b < hi) || (a <= lo && hi <= b))) continue;
      seq.push_back(&n->seq);
      if (a <= lo) w_dur.push_back(round6(sub(py_min(w.end, n->end), w.start)));
      else if (b >= hi) w_dur.push_back(round6(sub(w.end, py_max(w.start, n->start))));
      else w_dur.push_back(round6(n->dur));                   // unreachable in the reference too (covered by the first branch)
    }
    static const std::string rest = "rest";
    if (seq.size() == s0) {
      seq.push_back(&rest);
      w_dur.push_back(word_len);
    }
    const Num covered = round6(py_sum(w_dur, 0, w_dur.size()));
    if (covered.v < word_len.v) {
      seq.push_back(&rest);
      w_dur.push_back(sub(word_len, covered));
    }
    dur.insert(dur.end(), w_dur.begin(), w_dur.end());
  }
  seq_out->clear(), dur_out->clear();
  for (size_t i = 0; i < seq.size(); ++i) {
    if (i) *seq_out += ' ', *dur_out += ' ';
    *seq_out += *seq[i];
    *dur_out += py_str(round6(dur[i]));
  }
  return 0;
}

// Copies a field with its NUL when it fits; *size = its bytes including the NUL.
void give(const std::string& s, char* buf, size_t cap, size_t* size) {
  *size = s.size() + 1;
  if (buf && cap >= *size) memcpy(buf, s.c_str(), *size);
}

// The fields of one result (some_notes): chunk offsets begin / sample_rate, as some_notes_midi takes them.
int notes_fields(const some_notes* n, int sample_rate, double timestep, const char* ph_dur, const char* ph_num, bool round_midi,
                 std::string* seq, std::string* dur) {
  const int clips = some_notes_clips(n);
  if (clips < 0) return -1;
  std::vector<double> offsets(clips);
  std::vector<int32_t> counts(clips);
  std::vector<float> midi;
  std::vector<int32_t> frames;
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
    midi.insert(midi.end(), m, m + k), frames.insert(frames.end(), d, d + k), rest.insert(rest.end(), r, r + k);
  }
  std::vector<Note> notes;
  if (note_timeline(clips, offsets.data(), counts.data(), midi.data(), frames.data(), rest.data(), timestep, &notes)) return -1;
  return row_fields(notes, ph_dur, ph_num, round_midi, seq, dur);
}

// ---------------------------------------------------------------------------------------------- paths and files
// str(pathlib.PurePosixPath(p)): repeated slashes and '.' components dropped, no trailing slash, '' -> '.'.
std::string py_path(const std::string& p) {
  std::string root = p.rfind("//", 0) == 0 && p.rfind("///", 0) != 0 ? "//" : (p.rfind("/", 0) == 0 ? "/" : "");
  std::string out;
  size_t i = 0;
  while (i <= p.size()) {
    const size_t j = std::min(p.find('/', i), p.size());
    const std::string part = p.substr(i, j - i);
    if (!part.empty() && part != ".") out += (out.empty() ? "" : "/") + part;
    i = j + 1;
  }
  if (root.empty() && out.empty()) return ".";
  return root + out;
}
// str(PurePosixPath(a) / b): an absolute b replaces a.
std::string py_join(const std::string& a, const std::string& b) {
  if (!b.empty() && b[0] == '/') return py_path(b);
  return py_path(a.empty() ? b : a + "/" + b);
}

bool path_exists(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0;
}

int read_all(const std::string& path, std::vector<uint8_t>* out) {
  FILE* f = fopen(path.c_str(), "rb");
  SOME_REQUIRE(f != nullptr, "cannot open '%s': %s", path.c_str(), strerror(errno));
  struct stat st;                                             // one read of the whole file when its size is known
  out->resize(fstat(fileno(f), &st) == 0 && st.st_size > 0 ? static_cast<size_t>(st.st_size) : 0);
  size_t len = out->empty() ? 0 : fread(out->data(), 1, out->size(), f);
  out->resize(len);
  uint8_t chunk[1 << 16];
  for (size_t got; (got = fread(chunk, 1, sizeof(chunk), f)) > 0;) out->insert(out->end(), chunk, chunk + got);
  const bool bad = ferror(f) != 0;
  fclose(f);
  SOME_REQUIRE(!bad, "cannot read '%s'", path.c_str());
  return 0;
}

// ---------------------------------------------------------------------------------------------- the csv module
// repr() of a str, for DictWriter's message.
std::string py_str_repr(const std::string& s) {
  const bool dq = s.find('\'') != std::string::npos && s.find('"') == std::string::npos;
  const char q = dq ? '"' : '\'';
  std::string out(1, q);
  for (unsigned char ch : s) {
    if (ch == q || ch == '\\') out += '\\', out += static_cast<char>(ch);
    else if (ch == '\n') out += "\\n";
    else if (ch == '\r') out += "\\r";
    else if (ch == '\t') out += "\\t";
    else if (ch < 0x20 || ch == 0x7F) {
      char h[8];
      snprintf(h, sizeof(h), "\\x%02x", ch);
      out += h;
    } else {
      out += static_cast<char>(ch);
    }
  }
  return out + q;
}

bool valid_utf8(const std::string& s, size_t* bad) {
  const unsigned char* p = reinterpret_cast<const unsigned char*>(s.data());
  const size_t n = s.size();
  for (size_t i = 0; i < n;) {
    const unsigned c = p[i];
    int len;
    unsigned cp;
    if (c < 0x80) len = 1, cp = c;
    else if (c >= 0xC2 && c <= 0xDF) len = 2, cp = c & 0x1F;
    else if (c >= 0xE0 && c <= 0xEF) len = 3, cp = c & 0x0F;
    else if (c >= 0xF0 && c <= 0xF4) len = 4, cp = c & 0x07;
    else return *bad = i, false;
    if (i + len > n) return *bad = i, false;
    for (int k = 1; k < len; ++k) {
      if ((p[i + k] & 0xC0) != 0x80) return *bad = i, false;
      cp = cp << 6 | (p[i + k] & 0x3F);
    }
    if ((len == 3 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) || (len == 4 && (cp < 0x10000 || cp > 0x10FFFF)))
      return *bad = i, false;
    i += len;
  }
  return true;
}

// csv.reader(f) over a file opened with newline='': the excel dialect's state machine (_csv.c, strict off), fed line by line
// (lines end after \n, \r\n or a lone \r), an end-of-line event after each line; blank lines give [] (DictReader skips them).
constexpr long kFieldLimit = 131072;                          // csv.field_size_limit()
int csv_records(const std::string& text, std::vector<std::vector<std::string>>* records) {
  enum { START_RECORD, START_FIELD, IN_FIELD, IN_QUOTED_FIELD, QUOTE_IN_QUOTED_FIELD, EAT_CRNL } state = START_RECORD;
  std::vector<std::string> fields;
  std::string field;
  long field_len = 0;                                         // code points
  const int EOL = -1;
  auto save = [&]() {
    fields.push_back(field);
    field.clear(), field_len = 0;
  };
  auto put = [&](int c) -> bool {
    if ((c & 0xC0) != 0x80 && field_len++ >= kFieldLimit) return false;
    field += static_cast<char>(c);
    return true;
  };
  auto step = [&](int c) -> int {
    const bool nl = c == '\n' || c == '\r';
    switch (state) {
      case START_RECORD:
        if (c == EOL) break;
        if (nl) {
          state = EAT_CRNL;
          break;
        }
        state = START_FIELD;
        // fall through
      case START_FIELD:
        if (nl || c == EOL) save(), state = c == EOL ? START_RECORD : EAT_CRNL;
        else if (c == '"') state = IN_QUOTED_FIELD;
        else if (c == ',') save();
        else if (!put(c)) return -1;
        else state = IN_FIELD;
        break;
      case IN_FIELD:
        if (nl || c == EOL) save(), state = c == EOL ? START_RECORD : EAT_CRNL;
        else if (c == ',') save(), state = START_FIELD;
        else if (!put(c)) return -1;
        break;
      case IN_QUOTED_FIELD:
        if (c == EOL) break;
        if (c == '"') state = QUOTE_IN_QUOTED_FIELD;
        else if (!put(c)) return -1;
        break;
      case QUOTE_IN_QUOTED_FIELD:
        if (c == '"') {
          if (!put(c)) return -1;
          state = IN_QUOTED_FIELD;
        } else if (c == ',') {
          save(), state = START_FIELD;
        } else if (nl || c == EOL) {
          save(), state = c == EOL ? START_RECORD : EAT_CRNL;
        } else {
          if (!put(c)) return -1;
          state = IN_FIELD;
        }
        break;
      case EAT_CRNL:
        if (c == EOL) state = START_RECORD;
        break;                                                 // (lines end at \r or \n: nothing else can follow here)
    }
    return 0;
  };
  const size_t n = text.size();
  size_t i = 0;
  while (i < n) {                                             // one line per pass
    do {
      const unsigned char c = text[i++];
      if (step(c)) goto too_long;
      if (c == '\n' || (c == '\r' && !(i < n && text[i] == '\n'))) break;
    } while (i < n);
    if (step(EOL)) goto too_long;
    if (state == START_RECORD) records->push_back(fields), fields.clear();
  }
  if (!field.empty() || state == IN_QUOTED_FIELD) {           // end of data inside a record
    save();
    records->push_back(fields);
  }
  return 0;
too_long:
  SOME_REQUIRE(false, "field larger than field limit (%ld) in record %zu", kFieldLimit, records->size() + 1);
}

const char* const kFieldnames[6] = {"name", "ph_seq", "ph_dur", "ph_num", "note_seq", "note_dur"};
enum { F_NAME = 0, F_PH_SEQ, F_PH_DUR, F_PH_NUM, F_NOTE_SEQ, F_NOTE_DUR };

// A DictReader row, as the six fieldnames see it: a value, or None (a short row's padding, or a column the header lacks).
struct Row {
  std::string v[6];
  bool has[6];
};

// One field as csv.writer writes it with QUOTE_MINIMAL: quoted when it holds a delimiter, quote, \r or \n; quotes doubled.
void csv_field(std::string* out, const std::string& f) {
  if (f.find_first_of(",\"\r\n") == std::string::npos) {
    *out += f;
    return;
  }
  *out += '"';
  for (char ch : f) {
    if (ch == '"') *out += '"';
    *out += ch;
  }
  *out += '"';
}

// ---------------------------------------------------------------------------------------------- the dataset command
struct Item {
  size_t row;
  std::string path;
  std::vector<uint8_t> bytes;
  double seconds = 0;
};
struct Group {
  std::vector<Item> items;
  std::string error;
};

// Reads the files of `todo` in order and hands out groups of at most `budget` frames (1 + n / hop per item, n its samples at
// the model's rate; an item over the budget goes alone), one group ahead of the consumer.
class Reader {
 public:
  Reader(std::vector<Item> todo, int sr, int hop, long long budget)
      : todo_(std::move(todo)), sr_(sr), hop_(hop), budget_(budget), thread_([this] { run(); }) {}
  ~Reader() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
    }
    cv_.notify_all();
    thread_.join();
  }
  // false when the groups are done
  bool next(Group* g) {
    std::unique_lock<std::mutex> lk(mu_);
    cv_.wait(lk, [this] { return !ready_.empty() || done_; });
    if (ready_.empty()) return false;
    *g = std::move(ready_.front());
    ready_.pop_front();
    cv_.notify_all();
    return true;
  }

 private:
  bool hand(Group&& g) {
    std::unique_lock<std::mutex> lk(mu_);
    cv_.wait(lk, [this] { return ready_.empty() || stop_; });
    if (stop_) return false;
    ready_.push_back(std::move(g));
    cv_.notify_all();
    return true;
  }
  bool taken() {
    std::unique_lock<std::mutex> lk(mu_);
    cv_.wait(lk, [this] { return ready_.empty() || stop_; });
    return !stop_;
  }
  void run() {
    Group g;
    long long frames = 0;
    for (Item& it : todo_) {
      {
        std::lock_guard<std::mutex> lk(mu_);
        if (stop_) break;
      }
      if (read_all(it.path, &it.bytes)) {
        g.error = some_last_error();
        g.items.clear();
        hand(std::move(g));
        g = Group();
        break;
      }
      some_audio_meta m;
      long long n = 0;
      if (some_audio_info(it.bytes.data(), static_cast<long long>(it.bytes.size()), &m) == 0 && m.rate > 0) {
        long long native = m.frames;
        if (native == 0 && m.channels > 0) native = m.data_bytes / m.channels / 2;   // FLAC without a stated length: a guess
        n = static_cast<long long>(static_cast<double>(native) * sr_ / m.rate);
        it.seconds = static_cast<double>(m.frames) / m.rate;
      }
      const long long t = 1 + n / hop_;
      if (!g.items.empty() && frames + t > budget_) {
        if (!hand(std::move(g)) || !taken()) break;        // read on only while the consumer runs the group before
        g = Group(), frames = 0;
      }
      g.items.push_back(std::move(it));
      frames += t;
    }
    if (!g.items.empty()) hand(std::move(g));
    std::lock_guard<std::mutex> lk(mu_);
    done_ = true;
    cv_.notify_all();
  }

  std::vector<Item> todo_;
  const int sr_, hop_;
  const long long budget_;
  std::mutex mu_;
  std::condition_variable cv_;
  std::deque<Group> ready_;
  bool stop_ = false, done_ = false;
  std::thread thread_;                                        // last: starts after the members above exist
};

double since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace

extern "C" int some_label_write(int n_chunks, const double* offsets, const int32_t* counts, const float* note_midi,
                                const int32_t* note_dur, const uint8_t* note_rest, double timestep, const char* ph_dur,
                                const char* ph_num, int round_midi, char* seq_buf, size_t seq_cap, size_t* seq_size, char* dur_buf,
                                size_t dur_cap, size_t* dur_size) {
  SOME_REQUIRE(n_chunks >= 0 && (n_chunks == 0 || (offsets && counts)) && ph_dur && ph_num && seq_size && dur_size,
               "some_label_write: bad arguments");
  std::vector<Note> notes;
  std::string seq, dur;
  if (note_timeline(n_chunks, offsets, counts, note_midi, note_dur, note_rest, timestep, &notes) ||
      row_fields(notes, ph_dur, ph_num, round_midi != 0, &seq, &dur)) {
    set_error("some_label_write: %s", std::string(some_last_error()).c_str());
    return -1;
  }
  give(seq, seq_buf, seq_cap, seq_size);
  give(dur, dur_buf, dur_cap, dur_size);
  return 0;
}

extern "C" int some_notes_label(const some_notes* n, int sample_rate, double timestep, const char* ph_dur, const char* ph_num,
                                int round_midi, char* seq_buf, size_t seq_cap, size_t* seq_size, char* dur_buf, size_t dur_cap,
                                size_t* dur_size) {
  SOME_REQUIRE(n && sample_rate > 0 && ph_dur && ph_num && seq_size && dur_size, "some_notes_label: bad arguments");
  std::string seq, dur;
  if (notes_fields(n, sample_rate, timestep, ph_dur, ph_num, round_midi != 0, &seq, &dur)) {
    set_error("some_notes_label: %s", std::string(some_last_error()).c_str());
    return -1;
  }
  give(seq, seq_buf, seq_cap, seq_size);
  give(dur, dur_buf, dur_cap, dur_size);
  return 0;
}

extern "C" int some_session_label_dataset(some_session* s, const char* dataset_dir, const char* csv_path, int round_midi,
                                          int overwrite, const some_label_params* params, some_label_missing_fn on_missing,
                                          void* user, some_label_report* report) {
  const auto t0 = std::chrono::steady_clock::now();
  SOME_REQUIRE(dataset_dir != nullptr, "some_session_label_dataset: bad arguments");
  SOME_REQUIRE(!params || params->max_frames >= 0, "some_session_label_dataset: negative frame budget");
  const std::string data = py_path(dataset_dir);
  const std::string out_path = csv_path ? py_path(csv_path) : py_join(data, "transcriptions.csv");
  SOME_REQUIRE(overwrite || !path_exists(out_path),
               "some_session_label_dataset: The CSV path '%s' already exists. Please re-try with --overwrite option.", out_path.c_str());
  // read and check the table before any GPU work
  const std::string in_path = py_join(data, "transcriptions.csv");
  std::vector<uint8_t> raw;
  if (read_all(in_path, &raw)) return -1;
  const std::string text(raw.begin(), raw.end());
  size_t bad = 0;
  SOME_REQUIRE(valid_utf8(text, &bad), "some_session_label_dataset: '%s' is not UTF-8 (byte %zu)", in_path.c_str(), bad);
  std::vector<std::vector<std::string>> records;
  if (csv_records(text, &records)) {
    set_error("some_session_label_dataset: '%s': %s", in_path.c_str(), std::string(some_last_error()).c_str());
    return -1;
  }
  std::vector<std::string> header;
  size_t r0 = 0;
  if (!records.empty()) header = records[0], r0 = 1;
  std::vector<Row> rows;
  bool long_row0 = false, long_row = false;
  for (size_t r = r0; r < records.size(); ++r) {
    const std::vector<std::string>& rec = records[r];
    if (rec.empty()) continue;                                // DictReader skips blank lines
    Row row;
    for (int f = 0; f < 6; ++f) {
      long long col = -1;                                      // dict(zip(header, rec)): the last column of that name wins
      for (size_t k = 0; k < header.size(); ++k)
        if (header[k] == kFieldnames[f]) col = static_cast<long long>(k);
      row.has[f] = col >= 0 && static_cast<size_t>(col) < rec.size();    // short rows are padded with None
      if (row.has[f]) row.v[f] = rec[col];
    }
    if (rec.size() > header.size()) (rows.empty() ? long_row0 : long_row) = true;
    rows.push_back(row);
  }
  if (!rows.empty()) {
    for (int f : {F_NAME, F_PH_DUR, F_PH_NUM}) {
      bool found = false;
      for (const std::string& h : header) found |= h == kFieldnames[f];
      SOME_REQUIRE(found, "some_session_label_dataset: '%s' has no '%s' column", in_path.c_str(), kFieldnames[f]);
    }
    std::string wrong;                                         // DictWriter(extrasaction='raise'), at the first row
    for (size_t k = 0; k < header.size(); ++k) {
      bool known = false, seen = false;
      for (const char* f : kFieldnames) known |= header[k] == f;
      for (size_t j = 0; j < k; ++j) seen |= header[j] == header[k];
      if (!known && !seen) wrong += (wrong.empty() ? "" : ", ") + py_str_repr(header[k]);
    }
    if (long_row0 || (wrong.empty() && long_row)) wrong += wrong.empty() ? "None" : ", None";
    SOME_REQUIRE(wrong.empty(), "some_session_label_dataset: dict contains fields not in fieldnames: %s", wrong.c_str());
  }
  // the rows whose audio exists, and the warnings for the others, in row order
  std::vector<Item> todo;
  int64_t missing = 0;
  for (size_t r = 0; r < rows.size(); ++r) {
    const std::string name = rows[r].has[F_NAME] ? rows[r].v[F_NAME] : "None";
    const std::string wav = py_join(py_join(data, "wavs"), name + ".wav");
    if (!path_exists(wav)) {
      ++missing;
      if (on_missing) on_missing(wav.c_str(), user);
      continue;
    }
    for (int f : {F_PH_DUR, F_PH_NUM}) {
      SOME_REQUIRE(rows[r].has[f], "some_session_label_dataset: item '%s': no %s value", name.c_str(), kFieldnames[f]);
    }
    std::string seq, dur;                                      // the fields must parse before any GPU work
    std::vector<Note> none;
    if (row_fields(none, rows[r].v[F_PH_DUR].c_str(), rows[r].v[F_PH_NUM].c_str(), false, &seq, &dur)) {
      set_error("some_session_label_dataset: item '%s': %s", name.c_str(), std::string(some_last_error()).c_str());
      return -1;
    }
    Item it;
    it.row = r, it.path = wav;
    todo.push_back(std::move(it));
  }
  int64_t groups = 0, chunks = 0;
  double audio_seconds = 0, gpu_seconds = 0;
  const int64_t labelled = static_cast<int64_t>(todo.size());
  if (!todo.empty()) {
    SOME_REQUIRE(s != nullptr, "some_session_label_dataset: NULL session");
    some_session_info info;
    if (some_session_get_info(s, &info)) return -1;
    const long long budget =
        params && params->max_frames > 0 ? params->max_frames : SOME_SESSION_STEP_SAMPLES / info.hop;
    Reader reader(std::move(todo), info.sample_rate, info.hop, budget);
    std::vector<some_notes*> pool;
    struct Pool {
      std::vector<some_notes*>* p;
      ~Pool() {
        for (some_notes* n : *p) some_notes_destroy(n);
      }
    } pool_guard{&pool};
    Group g;
    while (reader.next(&g)) {
      SOME_REQUIRE(g.error.empty(), "some_session_label_dataset: %s", g.error.c_str());
      const int k = static_cast<int>(g.items.size());
      while (static_cast<int>(pool.size()) < k) {
        some_notes* n = nullptr;
        if (some_notes_create(&n)) return -1;
        pool.push_back(n);
      }
      std::vector<some_encoded> enc(k);
      for (int i = 0; i < k; ++i) enc[i] = {g.items[i].bytes.data(), static_cast<long long>(g.items[i].bytes.size())};
      const auto tg = std::chrono::steady_clock::now();
      const int rc = some_session_transcribe_encoded(s, enc.data(), k, params ? params->slicer : nullptr, pool.data());
      gpu_seconds += since(tg);
      if (rc) {
        const std::string msg = some_last_error();
        int i = -1, used = 0;
        if (sscanf(msg.c_str(), "some_session_transcribe_encoded: item %d%n", &i, &used) == 1 && i >= 0 && i < k) {
          const size_t at = msg.compare(used, 2, ": ") == 0 ? used + 2 : used;
          set_error("some_session_label_dataset: '%s': %s", g.items[i].path.c_str(), msg.c_str() + at);
        } else {
          set_error("some_session_label_dataset: %s", msg.c_str());
        }
        return -1;
      }
      ++groups;
      for (int i = 0; i < k; ++i) {
        Row& row = rows[g.items[i].row];
        const int clips = some_notes_clips(pool[i]);
        chunks += clips > 0 ? clips : 0;
        audio_seconds += g.items[i].seconds;
        if (notes_fields(pool[i], info.sample_rate, info.timestep, row.v[F_PH_DUR].c_str(), row.v[F_PH_NUM].c_str(),
                         round_midi != 0, &row.v[F_NOTE_SEQ], &row.v[F_NOTE_DUR])) {
          set_error("some_session_label_dataset: item '%s': %s", row.v[F_NAME].c_str(), std::string(some_last_error()).c_str());
          return -1;
        }
        row.has[F_NOTE_SEQ] = row.has[F_NOTE_DUR] = true;
      }
      g = Group();
    }
  }
  // DictWriter: the six fieldnames, QUOTE_MINIMAL, \r\n, '' for None
  std::string out;
  for (int f = 0; f < 6; ++f) out += (f ? "," : ""), out += kFieldnames[f];
  out += "\r\n";
  for (const Row& row : rows) {
    for (int f = 0; f < 6; ++f) {
      if (f) out += ',';
      if (row.has[f]) csv_field(&out, row.v[f]);
    }
    out += "\r\n";
  }
  FILE* f = fopen(out_path.c_str(), "wb");
  SOME_REQUIRE(f != nullptr, "some_session_label_dataset: cannot write '%s': %s", out_path.c_str(), strerror(errno));
  const bool written = fwrite(out.data(), 1, out.size(), f) == out.size();
  SOME_REQUIRE(fclose(f) == 0 && written, "some_session_label_dataset: cannot write '%s'", out_path.c_str());
  if (report) {
    report->rows = static_cast<int64_t>(rows.size());
    report->labelled = labelled;
    report->missing = missing;
    report->groups = groups;
    report->chunks = chunks;
    report->audio_seconds = audio_seconds;
    report->seconds = since(t0);
    report->gpu_seconds = gpu_seconds;
  }
  return 0;
}
