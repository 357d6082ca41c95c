"""CPU tests of the frame curves (some_notes_set_frames / some_notes_get_frames, csrc/session.cu): the refusals that need no
session, the ctypes prototypes against include/some_b200.h, and the example's option parsing.  The curves themselves, and
the refusal of notes filled with frames off, are tested on the GPU in tests/test_gpu_session_frames.py."""
import ctypes as C
import pathlib
import re
import subprocess

import pytest

from some_b200 import _lib
from some_b200 import session as nsess

REPO = pathlib.Path(__file__).resolve().parent.parent


def declaration(name):
    """The parameter list of `name` in the header, comments removed, as a list of C type strings."""
    header = re.sub(r'/\*.*?\*/', '', (REPO / 'include' / 'some_b200.h').read_text(), flags=re.S)
    m = re.search(r'\bint\s+' + name + r'\s*\(([^)]*)\)\s*;', header)
    assert m, name
    return [re.sub(r'\s+', ' ', p).strip() for p in m.group(1).split(',')]


def ctype_of(c_param):
    """The ctypes type a header parameter maps to: every pointer is passed as a pointer type, `int` as c_int."""
    base = re.sub(r'\b(const)\b', '', c_param).strip()
    stars = base.count('*')
    if stars == 0:
        assert base.split()[0] == 'int', c_param
        return C.c_int
    return 'pointer'


@pytest.mark.parametrize('name', ['some_notes_set_frames', 'some_notes_get_frames'])
def test_prototypes_match_the_header(name):
    restype, argtypes = _lib.EXPORTS[name]
    params = declaration(name)
    assert restype is C.c_int
    assert len(argtypes) == len(params), (params, argtypes)
    for p, a in zip(params, argtypes):
        want = ctype_of(p)
        if want == 'pointer':
            assert a is _lib._vp or issubclass(a, C._Pointer), (p, a)
        else:
            assert a is want, (p, a)
    # the output pointers of get_frames are, in order: frames (int *), then midi, rest, bound, note_index (pointers to the
    # curves' first elements)
    if name == 'some_notes_get_frames':
        assert [p.split()[-1].lstrip('*') for p in params] == ['n', 'clip', 'frames', 'midi', 'rest', 'bound', 'note_index']
        assert argtypes[2] is not _lib._vp and argtypes[2]._type_ is C.c_int


def test_refusals_without_a_session():
    lib = _lib.load()
    with pytest.raises(_lib.SomeB200Error, match='some_notes_set_frames: null pointer'):
        _lib.check(lib.some_notes_set_frames(None, 1))
    t = C.c_int(-7)
    p = C.c_void_p()
    with pytest.raises(_lib.SomeB200Error, match='some_notes_get_frames: null pointer'):
        _lib.check(lib.some_notes_get_frames(None, 0, C.byref(t), C.byref(p), None, None, None))
    n = nsess.Notes()
    try:
        for on in (False, True):
            n.set_frames(on)
            for clip in (0, -1, 5):
                with pytest.raises(_lib.SomeB200Error, match=f'some_notes_get_frames: clip {clip} out of range'):
                    _lib.check(lib.some_notes_get_frames(n.handle, clip, C.byref(t), C.byref(p), None, None, None))
            assert t.value == -7                 # nothing written
            assert n.curves() == [] and n.results(0.01) == ([], [])
    finally:
        n.close()


def test_example_takes_the_frames_option():
    example = REPO / 'examples' / 'some_stream'
    if not example.is_file():
        pytest.skip('examples/some_stream is built with the library')
    for args in (['--frames'], ['--frames', '--peek', '100'], ['--peek', '100', '--frames', 'model.somemodel']):
        run = subprocess.run([str(example)] + args, capture_output=True, text=True, timeout=60)
        assert run.returncode == 2 and '[--frames]' in run.stderr, (args, run.stderr)
    bad = subprocess.run([str(example), '--frames', '--peek', '0', 'm', '-'], capture_output=True, text=True, timeout=60)
    assert bad.returncode == 2 and 'positive number of milliseconds' in bad.stderr
