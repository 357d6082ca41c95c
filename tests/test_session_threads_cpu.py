"""CPU tests of the session's call statistics (csrc/session.cu, some_session_get_stats): the argument refusals, the struct
layout the Python binding mirrors, and the documented step bound.  The scheduling itself is tested on the GPU in
tests/test_gpu_session_threads.py."""
import ctypes as C
import pathlib
import re

from some_b200 import _lib

HEADER = pathlib.Path(__file__).resolve().parent.parent / 'include' / 'some_b200.h'


def test_stats_refuses_null_pointers():
    lib = _lib.load()
    st = _lib.SessionStats()
    assert lib.some_session_get_stats(None, C.byref(st)) != 0
    assert 'some_session_get_stats: null pointer' in lib.some_last_error().decode()
    assert lib.some_session_get_stats(C.c_void_p(1), None) != 0
    assert 'some_session_get_stats: null pointer' in lib.some_last_error().decode()


def test_stats_struct_matches_the_header():
    text = HEADER.read_text()
    body = re.search(r'typedef struct \{([^}]*)\} some_session_stats;', text).group(1)
    fields = re.findall(r'int64_t (\w+);', body)
    assert fields == [name for name, _ in _lib.SessionStats._fields_]
    assert C.sizeof(_lib.SessionStats) == 8 * len(fields)


def test_step_bound_is_64_recordings_of_30_s():
    m = re.search(r'#define SOME_SESSION_STEP_SAMPLES (\d+)LL', HEADER.read_text())
    assert int(m.group(1)) == 64 * 30 * 44100
