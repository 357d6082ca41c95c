"""CPU tests of the dataset labelling in csrc/label.cu (some_label_write, some_session_label_dataset's table handling) against
some_b200/batch.py, which tests/golden/host_rows.npz pins to the unmodified reference, and against Python's csv module."""
import csv
import ctypes as C
import io
import pathlib
import re
import sys

import numpy as np
import pytest

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / 'golden'))

from host_row_cases import TIMESTEP, fake_segments, make_dataset_rows  # noqa: E402
from some_b200 import _lib, batch  # noqa: E402
from some_b200.session import label_write  # noqa: E402

GOLD = np.load(HERE / 'golden' / 'host_rows.npz')
FIELDS = ['name', 'ph_seq', 'ph_dur', 'ph_num', 'note_seq', 'note_dur']


def with_frames(segments, timestep):
    """The segments with their durations as frames (note_dur = frames * timestep exactly, as the session gives them)."""
    out = []
    for sg in segments:
        frames = np.rint(np.asarray(sg['note_dur']) / timestep).astype(np.int32)
        np.testing.assert_array_equal(frames.astype(np.float64) * timestep, sg['note_dur'])
        out.append(dict(sg, note_frames=frames))
    return out


def python_fields(offsets, segments, ph_dur, ph_num, round_midi):
    return batch.row_notes(ph_dur, ph_num, batch.note_timeline(offsets, segments), round_midi)


# ---------------------------------------------------------------------------------------------- golden rows
@pytest.mark.parametrize('round_midi', [False, True])
def test_label_write_gives_reference_csv_bytes(round_midi):
    out = io.StringIO(newline='')
    writer = csv.DictWriter(out, fieldnames=FIELDS)
    writer.writeheader()
    rows = []
    for r in make_dataset_rows():
        row = {k: r[k] for k in ('name', 'ph_seq', 'ph_dur', 'ph_num')}
        if r['name'] != 'missing':
            offsets, segments = fake_segments(r['seed'])
            row['note_seq'], row['note_dur'] = label_write(offsets, with_frames(segments, TIMESTEP), TIMESTEP, row['ph_dur'],
                                                           row['ph_num'], round_midi)
        rows.append(row)
    writer.writerows(rows)
    assert out.getvalue().encode('utf8') == GOLD[f'csv_round{int(round_midi)}'].tobytes()


# ---------------------------------------------------------------------------------------------- fuzz
TIMESTEPS = (512 / 44100, 512 / 48000, 512 / 22050, 512 / 16000)


def fuzz_item(rng):
    """One random item: (offsets, segments with note_frames, timestep, ph_dur, ph_num)."""
    timestep = TIMESTEPS[int(rng.integers(len(TIMESTEPS)))]
    n_chunks = int(rng.integers(0, 5))
    offsets, segments, t = [], [], 0.0
    for _ in range(n_chunks):
        n = int(rng.integers(0, 9))                              # 0: an empty chunk
        frames = rng.integers(0, 80, size=n).astype(np.int32)    # 0: a note of no length
        kind = rng.random()
        if kind < 0.2:                                           # quantised model: integer-valued pitches
            midi = np.round(rng.uniform(40, 85, size=n)).astype(np.float32)
        elif kind < 0.45:                                        # cents at x.495 / x.505 / x.5 / x.29 (28.999... -> 28)
            base = rng.integers(40, 85, size=n).astype(np.float64)
            frac = rng.choice([0.495, 0.505, -0.495, -0.505, 0.5, -0.5, 0.29, -0.29, 0.005, -0.005], size=n)
            midi = (base + frac).astype(np.float32)
        else:
            midi = rng.uniform(40, 85, size=n).astype(np.float32)
        rest = rng.random(n) < 0.2
        r = rng.random()
        if r < 0.3:
            off = round(t * 50) * 882 / 44100                   # slicer offsets: multiples of the 20 ms hop
        elif r < 0.6:
            off = round(t * 128) / 128                           # multiples of 2^-7: ties at the 7th decimal
        else:
            off = t
        offsets.append(off)
        segments.append({'note_midi': midi, 'note_dur': frames.astype(np.float64) * timestep, 'note_rest': rest,
                         'note_frames': frames})
        t = off + float(frames.sum()) * timestep + float(rng.uniform(-0.4, 1.0))    # negative: overlapping chunks
        t = max(t, 0.0)
    # word edges: near note edges at exactly +-tolerance (decimal), random points, repeats (zero-length words)
    edges_src = []
    for off, sg in zip(offsets, segments):
        ends = off + np.cumsum(sg['note_dur'])
        edges_src.extend(ends.tolist())
    total = max([t] + edges_src + [0.5])
    edges = []
    for _ in range(int(rng.integers(1, 10))):
        r = rng.random()
        if edges_src and r < 0.4:
            e = float(rng.choice(edges_src)) + float(rng.choice([0.05, -0.05, 0.0, 0.049999, 0.050001]))
        elif edges and r < 0.5:
            e = edges[-1]                                        # a zero-length word
        else:
            e = float(rng.uniform(0, total))
        edges.append(max(e, 0.0))
    edges = sorted(edges)
    if rng.random() < 0.7:
        edges = [0.0] + edges
    spans = np.diff(np.concatenate([[0.0], edges])) if edges else np.array([])
    ph_dur, ph_num = [], []
    for w in spans:
        k = int(rng.integers(1, 4))
        cuts = np.sort(rng.uniform(0, w, size=k - 1)) if w > 0 else np.zeros(k - 1)
        parts = np.diff(np.concatenate([[0.0], cuts, [w]]))
        for p in parts:
            r = rng.random()
            if r < 0.55:
                s = f'{p:.6f}'
            elif r < 0.7:                                        # a 7th-decimal value, ties included, rounded by the reader
                s = f'{round(p * 1e6) / 1e6:.6f}' + str(int(rng.choice([5, 5, 1, 9])))
            elif r < 0.8:
                s = f'{p:.4e}'                                   # exponent form
            elif r < 0.9:
                s = f'{rng.uniform(0, 1e-4):.7f}'                # below 1e-4: 5e-05 in the output
            else:
                s = repr(round(float(p), 6))
            ph_dur.append(s)
        ph_num.append(k)
    if not ph_num or rng.random() < 0.15:
        ph_num.insert(int(rng.integers(0, len(ph_num) + 1)), 0)  # a word without phonemes
    if rng.random() < 0.05:
        ph_num.insert(0, 0)                                      # leading empty words: the int clock, "0"
    if not ph_dur:
        ph_dur = ['0.5']
    return offsets, segments, timestep, ' '.join(ph_dur), ' '.join(str(k) for k in ph_num)


def test_label_write_fuzz_equals_batch_py():
    rng = np.random.default_rng(20260)
    mismatches = []
    n_items = 20000
    for i in range(n_items):
        offsets, segments, timestep, ph_dur, ph_num = fuzz_item(rng)
        round_midi = bool(i % 2)
        want = python_fields(offsets, segments, ph_dur, ph_num, round_midi)
        got = label_write(offsets, segments, timestep, ph_dur, ph_num, round_midi)
        if got != want:
            mismatches.append((i, ph_dur, ph_num, want, got))
    assert not mismatches, mismatches[:3]


def test_fuzz_covers_the_traps():
    """The fuzz items reach the cases the restatement must get right."""
    rng = np.random.default_rng(20260)
    seen = {'tiny': 0, 'tie7': 0, 'zero_word': 0, 'int_word': 0, 'empty_chunk': 0, 'overlap': 0, 'quantised': 0}
    for _ in range(3000):
        offsets, segments, _, ph_dur, ph_num = fuzz_item(rng)
        toks = ph_dur.split(' ')
        seen['tiny'] += any(0 < float(x) < 1e-4 for x in toks)
        seen['tie7'] += any('.' in x and 'e' not in x and len(x.split('.')[1]) == 7 and x.endswith('5') for x in toks)
        seen['zero_word'] += ' 0' in ' ' + ph_num
        seen['int_word'] += ph_num.startswith('0')
        seen['empty_chunk'] += any(len(sg['note_frames']) == 0 for sg in segments)
        seen['quantised'] += any(len(sg['note_midi']) and np.all(sg['note_midi'] == np.round(sg['note_midi'])) for sg in segments)
        ends = [o + float(sg['note_dur'].sum()) for o, sg in zip(offsets, segments)]
        seen['overlap'] += any(o < e for o, e in zip(offsets[1:], ends[:-1]))
    assert all(v > 20 for v in seen.values()), seen


def test_compensated_sum_decides_the_field():
    """CPython 3.12's sum() is Neumaier-compensated; a plain left-to-right loop loses the word's last digit here."""
    ph_dur, ph_num = '10000000000 0.123456 -10000000000', '3'

    def plain(xs, start=0):
        for x in xs:
            start = start + x
        return start

    for round_midi in (False, True):
        want = python_fields([], [], ph_dur, ph_num, round_midi)
        assert want == ('rest', '0.123456')
        batch.sum = plain                                        # shadows the builtin inside batch.py
        try:
            assert python_fields([], [], ph_dur, ph_num, round_midi) == ('rest', '0.123455')
        finally:
            del batch.sum
        assert label_write([], [], TIMESTEP, ph_dur, ph_num, round_midi) == want


def test_rounding_repr_and_pitch_names():
    seg = {'note_midi': np.array([60.29, 60.495, 60.505, 61.5, 62.5, 59.71, 0.0, 127.0], np.float32),
           'note_rest': np.zeros(8, bool), 'note_frames': np.array([10, 3, 7, 1, 20, 5, 4, 9], np.int32)}
    seg['note_dur'] = seg['note_frames'] * TIMESTEP
    for ph_dur, ph_num in [('0.00005 0.0000005 2 0.1', '1 1 1 1'), ('0.0078125 0.0234375 1e-05 5E-5', '2 0 2'),
                           ('0.1 0.2 0.3 0.4 0.5 0.6', '6'), ('1 .5 5. +0.25', '0 0 4')]:
        for round_midi in (False, True):
            want = python_fields([0.0], [seg], ph_dur, ph_num, round_midi)
            assert label_write([0.0], [seg], TIMESTEP, ph_dur, ph_num, round_midi) == want
    seq, _ = label_write([0.0], [seg], TIMESTEP, '1', '1', False)
    assert batch.calc_seq(float(np.float32(60.29)), False) == 'C4+28'            # int() truncates 28.999...
    assert 'C4+28' in seq
    assert label_write([], [], TIMESTEP, '0.00005', '1', True) == ('rest', '5e-05')
    assert label_write([], [], TIMESTEP, '2', '1', True) == ('rest', '2.0')
    assert label_write([], [], TIMESTEP, '0.5', '0 1', True) == ('rest rest', '0 0.5')


@pytest.mark.parametrize('field,bad', [('ph_dur', ''), ('ph_dur', 'inf'), ('ph_dur', 'nan'), ('ph_dur', '1_0'),
                                       ('ph_dur', '0.5  0.5'), ('ph_dur', '0x10'), ('ph_dur', '.'), ('ph_dur', '1e'),
                                       ('ph_num', '1.0'), ('ph_num', ''), ('ph_num', 'a')])
def test_malformed_fields_are_refused(field, bad):
    args = {'ph_dur': '0.5', 'ph_num': '1'}
    args[field] = bad
    with pytest.raises(_lib.SomeB200Error, match=field):
        label_write([], [], TIMESTEP, args['ph_dur'], args['ph_num'], False)


def test_label_write_sizes():
    lib = _lib.load()
    seq_n, dur_n = C.c_size_t(), C.c_size_t()
    assert lib.some_label_write(0, None, None, None, None, None, TIMESTEP, b'0.5 0.25', b'1 1', 0, None, 0, C.byref(seq_n), None, 0,
                                C.byref(dur_n)) == 0
    assert (seq_n.value, dur_n.value) == (len('rest rest') + 1, len('0.5 0.25') + 1)
    small = C.create_string_buffer(4)
    assert lib.some_label_write(0, None, None, None, None, None, TIMESTEP, b'0.5 0.25', b'1 1', 0, small, 4, C.byref(seq_n), None,
                                0, C.byref(dur_n)) == 0
    assert small.raw == b'\0' * 4                                # too small: untouched


# ---------------------------------------------------------------------------------------------- the table (no audio: no GPU)
def run_native(dataset, csv_path=None, overwrite=False):
    """some_session_label_dataset without a session: possible while no row has an audio file."""
    lib = _lib.load()
    seen = []
    cb = _lib.LABEL_MISSING_FN(lambda p, _u: seen.append(p.decode('utf8')))
    rep = _lib.LabelReport()
    rc = lib.some_session_label_dataset(None, str(dataset).encode(), None if csv_path is None else str(csv_path).encode(), 0,
                                        int(overwrite), None, cb, None, C.byref(rep))
    if rc:
        raise _lib.SomeB200Error(lib.some_last_error().decode('utf8'))
    return seen, rep


def run_python(dataset, csv_path=None, overwrite=False, capsys=None):
    batch.batch_infer_dataset(dataset, None, {'audio_sample_rate': 44100}, csv=csv_path, overwrite=overwrite)
    out = capsys.readouterr().out
    return re.findall(r"WARNING: audio file does not exist: '(.*?)'\n(?=WARNING|$)", out, re.S)


TABLES = {
    'plain': 'name,ph_seq,ph_dur,ph_num\nitem0,a b,0.1 0.2,2\nitem1,a,0.5,1\n',
    'quoted': ('name,ph_seq,ph_dur,ph_num,note_seq,note_dur\r\n"a,b","x ""y"" z",0.1,1,C4,0.1\r\n'
               '"multi\nline",a,"0.2",1\r\n"cr\rname",a,0.3,1,,\r\n'),
    'unicode_short_blank': 'name,ph_seq,ph_dur,ph_num,note_seq\n\nちょう,a,0.1,1\nshort\n\n\nx,"",,\n"é",b\n',
    'cr_only': 'name,ph_seq,ph_dur,ph_num\ra,b,0.1,1\rc,d,0.2,1',
    'odd_quotes': 'name,ph_seq,ph_dur,ph_num\nab"c,"q"x,0.1,1\n"open,still\nopen',
    'reordered_dup': 'ph_num,ph_dur,name,name,ph_seq\n1,0.1,first,second,a\n2,0.2,only\n',
    'header_only': 'name,ph_seq,ph_dur,ph_num\n',
    'empty': '',
    'slashes': 'name,ph_seq,ph_dur,ph_num\nsub/dir,a,0.1,1\n./dot,a,0.1,1\n/abs/x,a,0.1,1\n',
}


@pytest.mark.parametrize('table', sorted(TABLES))
def test_table_round_trip_equals_csv_module(tmp_path, capsys, table):
    ds = tmp_path / 'ds'
    (ds / 'wavs').mkdir(parents=True)
    (ds / 'transcriptions.csv').write_bytes(TABLES[table].encode('utf8'))
    want_missing = run_python(ds, tmp_path / 'py.csv', capsys=capsys)
    got_missing, rep = run_native(ds, tmp_path / 'c.csv')
    assert (tmp_path / 'c.csv').read_bytes() == (tmp_path / 'py.csv').read_bytes()
    assert got_missing == want_missing
    assert rep.missing == len(want_missing) and rep.labelled == 0 and rep.rows == len(want_missing)


def test_default_output_and_overwrite(tmp_path, capsys):
    ds = tmp_path / 'ds'
    (ds / 'wavs').mkdir(parents=True)
    src = TABLES['quoted'].encode('utf8')
    (ds / 'transcriptions.csv').write_bytes(src)
    (tmp_path / 'py').mkdir()
    (tmp_path / 'py' / 'wavs').mkdir()
    (tmp_path / 'py' / 'transcriptions.csv').write_bytes(src)
    run_python(tmp_path / 'py', overwrite=True, capsys=capsys)
    run_native(str(ds) + '/', overwrite=True)
    assert (ds / 'transcriptions.csv').read_bytes() == (tmp_path / 'py' / 'transcriptions.csv').read_bytes()


def refusal_cases(tmp_path):
    yield 'exists', 'name,ph_seq,ph_dur,ph_num\na,b,0.1,1\n', False
    yield 'no_name', 'nam,ph_seq,ph_dur,ph_num\na,b,0.1,1\n', True
    yield 'no_ph_dur', 'name,ph_seq,ph_num\na,b,1\n', True
    yield 'no_ph_num', 'name,ph_seq,ph_dur\na,b,0.1\n', True
    yield 'extra_column', 'name,ph_seq,ph_dur,ph_num,speaker\na,b,0.1,1,x\n', True
    yield 'long_row', 'name,ph_seq,ph_dur,ph_num\na,b,0.1,1,extra\n', True
    yield 'not_utf8', 'name,ph_seq,ph_dur,ph_num\n\udcff,b,0.1,1\n', True


@pytest.mark.parametrize('case', ['exists', 'no_name', 'no_ph_dur', 'no_ph_num', 'extra_column', 'long_row', 'not_utf8'])
def test_refusals_leave_the_output_untouched(tmp_path, case):
    text, overwrite = {c: (t, o) for c, t, o in refusal_cases(tmp_path)}[case]
    ds = tmp_path / 'ds'
    (ds / 'wavs').mkdir(parents=True)
    (ds / 'transcriptions.csv').write_bytes(text.encode('utf8', 'surrogateescape'))
    out = tmp_path / 'out.csv'
    before = b'previous output\r\n\x00\xff'
    out.write_bytes(before)
    with pytest.raises(_lib.SomeB200Error) as e:
        run_native(ds, out, overwrite=overwrite)
    assert out.read_bytes() == before
    msg = str(e.value)
    if case == 'exists':
        with pytest.raises(FileExistsError) as pe:
            batch.batch_infer_dataset(ds, None, {'audio_sample_rate': 44100}, csv=out)
        assert str(pe.value) in msg
    elif case == 'extra_column':
        assert "dict contains fields not in fieldnames: 'speaker'" in msg
    elif case == 'long_row':
        assert 'dict contains fields not in fieldnames: None' in msg
    elif case == 'not_utf8':
        assert 'UTF-8' in msg
    else:
        assert f"no '{case[3:]}' column" in msg


def test_unparsable_fields_refused_before_any_work(tmp_path):
    ds = tmp_path / 'ds'
    (ds / 'wavs').mkdir(parents=True)
    (ds / 'wavs' / 'b.wav').write_bytes(b'not read before the refusal')
    (ds / 'transcriptions.csv').write_text('name,ph_seq,ph_dur,ph_num\na,x,bad,1\nb,y,0.1 oops,2\n', encoding='utf8')
    with pytest.raises(_lib.SomeB200Error, match="item 'b'.*ph_dur value 1 'oops'"):
        run_native(ds, tmp_path / 'out.csv')
    assert not (tmp_path / 'out.csv').exists()
    (ds / 'transcriptions.csv').write_text('name,ph_seq,ph_dur,ph_num\nb,y,0.1 0.2,2\n', encoding='utf8')
    with pytest.raises(_lib.SomeB200Error, match='NULL session'):  # a row with audio needs a session
        run_native(ds, tmp_path / 'out.csv')
    assert not (tmp_path / 'out.csv').exists()
