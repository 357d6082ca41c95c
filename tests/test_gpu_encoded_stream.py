"""Encoded streams on the H100 (some_stream_open_encoded, some_stream_push_bytes*, csrc/session.cu): a WAV or FLAC file pushed
as its bytes arrive, split in any way, gives chunk by chunk exactly what some_session_transcribe_encoded gives for the whole
file, in the push where a PCM stream fed the samples decoded in each push would deliver them; many streams in one call equal
each stream alone; refusals come with the encoded call's message; the bytes held stay within a frame and a push."""
import pathlib
import subprocess
import threading

import numpy as np
import pytest

from oracle import flac as of
from some_b200 import _lib, audio, export, synth
from some_b200 import session as nsess

import test_gpu_encoded as ge

pytestmark = pytest.mark.gpu
REPO = pathlib.Path(__file__).resolve().parent.parent


@pytest.fixture(scope='module', params=['two_head', 'quant_two_head'])
def sess(request, tmp_path_factory):
    d = tmp_path_factory.mktemp(request.param)
    path = export.export(synth.write_checkpoint(d, synth.named_config(request.param), seed=1234))
    s = nsess.Session(path, 0)
    s.kind, s.path = request.param, path
    yield s
    s.close()


def var_blocks(n):
    sizes = []
    while sum(sizes) < n:
        sizes.append(min([4096, 1152, 577][len(sizes) % 3], n - sum(sizes)))
    return sizes


def mono(seed, seconds, rate):
    return synth.synth_waveform(seed, seconds=seconds, sr=rate, silence_gaps=True) * np.float32(0.9)


FILES = {   # name: the file's bytes (60-90 s with silence gaps)
    'wav_u8_1ch_44k': lambda: ge.wav_file(mono(31, 62.0, 44100), 44100, 'u8'),
    'wav_s16_2ch_48k': lambda: ge.wav_file(ge.stereo(32, 75.0, 48000), 48000, 's16'),
    'wav_s24_12ch_22k': lambda: ge.wav_file(mono(33, 60.0, 22050)[:, None] * np.linspace(0.3, 1.0, 12, dtype=np.float32), 22050,
                                            's24'),                     # one silence pattern: the down-mix keeps its gaps
    'wav_s32_1ch_48k': lambda: ge.wav_file(mono(34, 64.0, 48000), 48000, 's32'),
    'wav_f32_2ch_22k': lambda: ge.wav_file(ge.stereo(35, 70.0, 22050), 22050, 'f32'),
    'wav_f64_2ch_44k': lambda: ge.wav_file(ge.stereo(36, 60.0, 44100), 44100, 'f64'),
    'flac_16_fixed_44k_id3': lambda: ge.flac_file(mono(37, 90.0, 44100), 44100, 16, id3=of.id3_tag()),
    'flac_24_variable_midside_48k': lambda: ge.flac_file(ge.stereo(38, 66.0, 48000), 48000, 24, channel_mode='mid_side',
                                                         variable=True, blocksize=var_blocks(66 * 48000)),
    'flac_16_unknown_length_22k': lambda: ge.flac_file(ge.stereo(39, 61.0, 22050), 22050, 16, total_samples=0,
                                                       channel_mode='left_side'),
}


@pytest.fixture(scope='module')
def files():
    return {name: make() for name, make in FILES.items()}


def byte_sizes(n, rng, small=1500):
    """Single bytes over the header, then random sizes from 1 byte to 256 KB."""
    sizes = [1] * min(small, n)
    while sum(sizes) < n:
        sizes.append(int(rng.integers(1, 1 << 18)))
    return sizes


def push_all(st, data, sizes, infos=None):
    """Every push's chunks, then the finish's: [(ranges, notes)] per call."""
    out, a = [], 0
    for m in sizes:
        _, r, nt = st.push(data[a:a + m])
        a += m
        out.append((r, nt))
        if infos is not None:
            infos.append(st.info()['received'])
    _, r, nt = st.finish()
    out.append((r, nt))
    return out


def flatten(calls):
    ranges, notes = [], []
    for r, nt in calls:
        ranges += r
        notes += nt
    return ranges, notes


@pytest.mark.parametrize('name', list(FILES))
def test_stream_equals_transcribe_encoded(sess, files, name, tmp_path):
    data = files[name]
    _, want_ranges, want_notes = sess.transcribe_encoded([data])[0]
    rng = np.random.default_rng(len(name))
    sizes = byte_sizes(len(data), rng)
    infos = []
    with sess.stream_encoded() as st:
        calls = push_all(st, data, sizes, infos)
        meta = st.meta()
        assert meta['bytes_received'] == len(data)
    ranges, notes = flatten(calls)
    assert ranges == want_ranges
    ge.assert_same_notes(notes, want_notes)
    assert sum(len(r) for r, _ in calls[:-1]) >= 2, 'several chunks arrive before the finish'
    assert meta['rate'] == audio.load(_write(tmp_path, name, data), sr=None)[1]
    # the same chunks, in the same pushes, as a PCM stream fed the samples each push decoded
    if name in ('wav_s16_2ch_48k', 'flac_24_variable_midside_48k', 'flac_16_fixed_44k_id3'):
        y, rate = audio.load(_write(tmp_path, name, data), sr=None)
        prev, pcm_calls = 0, []
        with sess.stream(rate) as ps:
            for got in infos:
                _, r, nt = ps.push(y[prev:got])
                pcm_calls.append((r, nt))
                prev = got
            _, r, nt = ps.finish()
            pcm_calls.append((r, nt))
        assert len(pcm_calls) == len(calls)
        for (pr, pn), (r, nt) in zip(pcm_calls, calls):
            assert pr == r
            ge.assert_same_notes(pn, nt)


def _write(tmp_path, name, data):
    p = tmp_path / (name + ('.flac' if name.startswith('flac') else '.wav'))
    p.write_bytes(data)
    return p


def test_whole_file_in_one_push_and_byte_by_byte_header(sess, files):
    for name in ('wav_s24_12ch_22k', 'flac_16_unknown_length_22k'):
        data = files[name]
        _, want_ranges, want_notes = sess.transcribe_encoded([data])[0]
        for sizes in ([len(data)], [1] * 5000 + [len(data) - 5000]):
            with sess.stream_encoded() as st:
                ranges, notes = flatten(push_all(st, data, sizes))
            assert ranges == want_ranges
            ge.assert_same_notes(notes, want_notes)


def test_push_bytes_many_equals_each_stream_alone(sess, files):
    names = list(FILES) * 2
    names = names[:16]
    datas = [files[n] for n in names]
    want = [r[1:] for r in sess.transcribe_encoded(datas)]
    rng = np.random.default_rng(7)
    streams = [sess.stream_encoded() for _ in names]
    got = [([], []) for _ in names]
    pos = [0] * len(names)
    done = [False] * len(names)
    tick = 0
    while not all(done):
        items, fin, idx = [], [], []
        for i, st in enumerate(streams):
            if done[i]:
                continue
            m = int(rng.integers(0, 1 << 17)) if tick else 300
            chunk = datas[i][pos[i]:pos[i] + m]
            pos[i] += len(chunk)
            f = pos[i] >= len(datas[i]) and rng.random() < 0.5
            items.append((st, chunk))
            fin.append(f)
            idx.append(i)
        for i, (_, r, nt) in zip(idx, sess.push_bytes_many(items, fin)):
            got[i][0].extend(r)
            got[i][1].extend(nt)
        for i, f in zip(idx, fin):
            done[i] = done[i] or f
        tick += 1
    for st in streams:
        st.close()
    for (gr, gn), (wr, wn) in zip(got, want):
        assert gr == wr
        ge.assert_same_notes(gn, wn)


def test_threads_on_disjoint_streams(sess, files):
    names = ['wav_s16_2ch_48k', 'flac_16_fixed_44k_id3', 'wav_f32_2ch_22k']
    want = {n: sess.transcribe_encoded([files[n]])[0][1:] for n in names}
    got, errors = {}, []

    def run(n):
        try:
            with sess.stream_encoded() as st:
                got[n] = flatten(push_all(st, files[n], byte_sizes(len(files[n]), np.random.default_rng(3), small=10)))
        except Exception as e:          # noqa: BLE001 (reported below)
            errors.append(e)

    ts = [threading.Thread(target=run, args=(n,)) for n in names]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors
    for n in names:
        assert got[n][0] == want[n][0]
        ge.assert_same_notes(got[n][1], want[n][1])


def max_frame(flac: bytes) -> int:
    """STREAMINFO's largest frame in bytes."""
    si = flac.index(b'fLaC') + 8
    return int.from_bytes(flac[si + 7:si + 10], 'big')


def frame_ends(flac: bytes, count: int):
    """The end of each of the first `count` frames (oracle.flac's frame walk)."""
    info = of.parse_metadata(flac)
    buf = np.frombuffer(flac, np.uint8)
    out = np.zeros((info['channels'], max(info['max_blocksize'], 1)), np.int64)
    pos, ends = info['audio_offset'], []
    for _ in range(count):
        st, end, *_ = of._frame(buf, pos, len(flac), info['channels'], info['bps'], info['max_blocksize'], out, of.CRC8_T,
                                of.CRC16_T)
        assert st == of.OK
        ends.append(end)
        pos = end
    return ends


def corrupt_frame(flac: bytes, k: int):
    """The file with frame k's CRC-16 flipped (its parse is fine up to its last byte), and that frame's end."""
    end = frame_ends(flac, k + 1)[k]
    bad = bytearray(flac)
    bad[end - 1] ^= 0x10
    return bytes(bad), end


def _refusal(fn):
    with pytest.raises(_lib.SomeB200Error) as e:
        fn()
    return str(e.value)


def test_refusals(sess, files):
    flac = files['flac_16_fixed_44k_id3']
    m = audio.parse_flac(flac)
    # a flipped byte in frame 10's CRC-16: refused at the push that completes that frame, with the encoded call's text
    bad, end = corrupt_frame(flac, 10)
    reason = _refusal(lambda: sess.transcribe_encoded([bad])).split('item 0: ', 1)[1]
    assert 'CRC-16 mismatch' in reason
    with sess.stream_encoded() as st:
        a, msg = 0, None
        while msg is None:
            try:
                st.push(bad[a:a + 1000])
            except _lib.SomeB200Error as e:
                msg = str(e)
            a += 1000
        assert msg.endswith('some_stream_push_bytes: ' + reason) and a - 1000 < end <= a
        st.info(), st.meta()
        assert 'refused' in _refusal(lambda: st.push(b'x'))
    # cut mid-frame: refused at the finish
    cut = flac[:m.audio_offset + 70001]
    reason = _refusal(lambda: sess.transcribe_encoded([cut])).split('item 0: ', 1)[1]
    with sess.stream_encoded() as st:
        st.push(cut)
        assert _refusal(st.finish).endswith('some_stream_finish: ' + reason)
    # other containers (at the push that makes the refusal certain), an unsupported rate (at the push that completes the header)
    for data in (b'OggS' + bytes(60), b'ID3\x04\x00\x00\x00\x00\x00\x02ab' + bytes(40), b'\xff\xfb\x90\x00' + bytes(60)):
        reason = _refusal(lambda: sess.transcribe_encoded([data])).split('item 0: ', 1)[1]
        with sess.stream_encoded() as st:
            st.push(data[:4])
            assert _refusal(lambda: st.push(data[4:])).endswith('some_stream_push_bytes: ' + reason)
    fast = ge.wav_file(np.zeros(1000, np.float32), 1000000, 's16')
    reason = _refusal(lambda: sess.transcribe_encoded([fast])).split('item 0: ', 1)[1]
    with sess.stream_encoded() as st:
        assert _refusal(lambda: st.push(fast[:44])).endswith(reason)
    # the kinds of stream do not mix
    lib = sess.lib
    with sess.stream_encoded() as enc, sess.stream(44100) as pcm:
        assert 'encoded stream' in _refusal(lambda: _lib.check(lib.some_stream_push(enc.handle, None, 0, enc.notes.handle)))
        assert 'encoded stream' in _refusal(lambda: sess.push_many([(enc, np.zeros(10, np.float32))]))
        assert 'PCM stream' in _refusal(lambda: _lib.check(lib.some_stream_push_bytes(pcm.handle, b'RIFF', 4, pcm.notes.handle)))
        assert 'PCM stream' in _refusal(lambda: sess.push_bytes_many([(pcm, b'RIFF')]))
        assert 'PCM stream' in _refusal(lambda: _lib.check(lib.some_stream_get_meta(pcm.handle, _lib.AudioMeta(), None, None)))


def test_many_call_content_refusal_keeps_the_other_streams(sess, files):
    """One corrupt FLAC among healthy streams: the call raises StreamRefused with every item's results, and the healthy
    streams' chunks, concatenated over all calls, still equal transcribe_encoded."""
    bad, _ = corrupt_frame(files['flac_16_fixed_44k_id3'], 40)
    names = ['wav_s16_2ch_48k', 'flac_24_variable_midside_48k', 'wav_u8_1ch_44k']
    datas = [files[n] for n in names] + [bad]
    want = [r[1:] for r in sess.transcribe_encoded(datas[:3])]
    streams = [sess.stream_encoded() for _ in datas]
    got = [([], []) for _ in datas]
    live, pos, refused = list(range(len(datas))), [0] * len(datas), []
    block = 96000
    while live:
        items = [(streams[i], datas[i][pos[i]:pos[i] + block]) for i in live]
        fin = [pos[i] + block >= len(datas[i]) for i in live]
        try:
            res = sess.push_bytes_many(items, fin)
        except _lib.StreamRefused as e:
            assert f'stream {live.index(3)}: FLAC frame at byte offset' in str(e) and 'CRC-16 mismatch' in str(e)
            res = e.results
            refused.append(3)
            assert res[live.index(3)][1] == []
        for i, (_, r, nt) in zip(live, res):
            got[i][0].extend(r)
            got[i][1].extend(nt)
        for i in live:
            pos[i] += block
        live = [i for i, f in zip(live, fin) if not f and i not in refused]
    assert refused
    for (gr, gn), (wr, wn) in zip(got[:3], want):
        assert gr == wr
        ge.assert_same_notes(gn, wn)
    assert 'refused' in _refusal(lambda: sess.push_bytes_many([(streams[3], b'x')]))
    for st in streams:
        st.close()


def test_c_example_reads_encoded_bytes_from_stdin(sess, files):
    """examples/some_stream MODEL - prints, for a WAV and a FLAC byte stream, the lines formatted from transcribe_encoded."""
    if sess.kind != 'two_head':
        pytest.skip('one model kind is enough for the example')
    example = REPO / 'examples' / 'some_stream'
    for name in ('wav_s16_2ch_48k', 'flac_24_variable_midside_48k'):
        offsets, _, notes = sess.transcribe_encoded([files[name]])[0]
        want = ['%.17g %.9g %.17g %d' % (o, float(m), float(d), int(r))
                for o, nt in zip(offsets, notes) for m, d, r in zip(nt['note_midi'], nt['note_dur'], nt['note_rest'])]
        run = subprocess.run([str(example), str(sess.path), '-'], input=files[name], capture_output=True, timeout=300)
        assert run.returncode == 0, run.stderr
        lines = run.stdout.decode().splitlines()
        assert len(lines) > 20 and lines == want
    run = subprocess.run([str(example), str(sess.path), '-'], input=b'OggS' + bytes(100), capture_output=True, timeout=300)
    assert run.returncode == 1 and b'Ogg' in run.stderr


def test_many_call_argument_errors_change_no_stream(sess, files):
    a, b = sess.stream_encoded(), sess.stream_encoded()
    data = files['wav_s16_2ch_48k']
    sess.push_bytes_many([(a, data[:5000]), (b, data[:3000])])
    before = [(s.info(), s.meta()) for s in (a, b)]
    assert 'appears twice' in _refusal(lambda: sess.push_bytes_many([(a, data[5000:6000]), (a, data[5000:6000])]))
    c = sess.stream_encoded()
    with sess.stream(44100) as pcm:
        assert 'PCM stream' in _refusal(lambda: sess.push_bytes_many([(a, data[5000:6000]), (pcm, b'x')]))
    assert [(s.info(), s.meta()) for s in (a, b)] == before
    for s in (a, b, c):
        s.close()


def test_memory_stays_within_a_frame_and_a_push(sess):
    """A 10-minute FLAC with a 4 MB PICTURE block and a long leading silence: the host holds at most one frame plus the push,
    the device no more than a PCM stream of the same samples."""
    rate = 44100
    x = mono(41, 480.0, rate)
    x = np.concatenate([np.zeros(rate * 120, np.float32), x])
    data = ge.flac_file(x, rate, 16, blocksize=4096, metadata=[('PICTURE', bytes(4 << 20))])
    x = (np.clip(np.round(x * 32768), -32768, 32767) / 32768).astype(np.float32)   # the decoded samples
    frame_max = max_frame(data)
    push = 20000
    most, held_pcm = 0, 0
    with sess.stream_encoded() as st, sess.stream(rate) as ps:
        a, prev = 0, 0
        while a < len(data):
            st.push(data[a:a + push])
            a += push
            most = max(most, st.meta()['bytes_held'])
            got = st.info()['received']
            ps.push(x[prev:got])
            prev = got
            assert st.info()['held'] == ps.info()['held']
            held_pcm = max(held_pcm, ps.info()['held'])
        st.finish()
    assert most <= frame_max + push + 64, (most, frame_max)
