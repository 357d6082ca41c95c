"""Audio already on the GPU (csrc/downmix.cu, some_session_transcribe_device, some_stream_push_device*): the down-mix is
np.mean(y, axis=0) of librosa's (channels, n) view bit for bit in every layout, and the session, its streams and
batch.transcribe_recordings give from CUDA tensors exactly what they give from the host down-mix."""
import ctypes as C
import threading
import time

import numpy as np
import pytest
import torch

from some_b200 import _lib, audio, batch, export, plugin, synth
from some_b200 import session as nsess

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


@pytest.fixture(scope='module')
def ckpt(tmp_path_factory):
    return synth.write_checkpoint(tmp_path_factory.mktemp('two_head'), synth.named_config('two_head'), seed=1234)


@pytest.fixture(scope='module')
def path(ckpt):
    return export.export(ckpt)


@pytest.fixture(scope='module')
def sess(path):
    s = nsess.Session(path, 0)
    yield s
    s.close()


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def layout_copy(t: torch.Tensor) -> np.ndarray:
    """The host copy of a recording tensor with its layout's memory order: what numpy's mean reduces."""
    y = t.detach().cpu().numpy()
    if t.dim() == 1:
        return y
    ch, n = t.shape
    if n > 1 and t.stride(0) == 1 and t.stride(1) == ch:
        return np.ascontiguousarray(y.T).T             # [C, n] view of [n, C]
    return np.ascontiguousarray(y)


def host_mean(t: torch.Tensor) -> np.ndarray:
    y = layout_copy(t)
    return y if y.ndim == 1 else np.mean(y, axis=0)


def adversarial(rng, ch: int, n: int) -> np.ndarray:
    y = (rng.standard_normal((ch, n)) * 10.0 ** rng.integers(-38, 38, (ch, n))).astype(np.float32)
    k = max(n // 8, 1)
    y[:, :k] = rng.standard_normal((ch, 1)).astype(np.float32) * np.float32(1e30)
    if ch > 1:
        y[-1, :k] = -y[:-1, :k].sum(axis=0, dtype=np.float32)
    y[:, k:k + 3] = -0.0
    return y


def planar(y: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(y)).to(DEV)


def interleaved(y: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(y.T)).to(DEV).t()


def wide(y: np.ndarray, pad: int = 37) -> torch.Tensor:
    """A planar view with a storage offset and a channel stride larger than its frames."""
    ch, n = y.shape
    big = torch.zeros(ch + 1, n + 2 * pad, device=DEV)
    big[1:, pad:pad + n] = torch.from_numpy(y).to(DEV)
    return big[1:, pad:pad + n]


# --------------------------------------------------------------------------- the kernel
def test_downmix_is_numpys_mean_in_every_layout_and_at_tile_edges():
    rng = np.random.default_rng(5)
    tensors = []
    for n in (0, 1, 2, 1023, 1024, 1025, 3 * 1024 + 1):
        tensors.append(planar(adversarial(rng, 1, max(n, 1))[:, :n])[0])                      # mono [n]
    for ch in (1, 2, 3, 6, 8, 9, 16, 17, 128):
        per = 8192 // ch                                                                      # an interleaved tile
        for n in (1, 2, 1023, 1025, per - 1, per, per + 1, 2 * per + 1):
            y = adversarial(rng, ch, n)
            tensors += [planar(y), interleaved(y), wide(y)]
        tensors.append(wide(adversarial(rng, ch, 9))[:, 4:5])                                 # one strided frame
    tensors.append(wide(adversarial(rng, 2, 50000)))
    starts = np.concatenate([[0], np.cumsum([t.shape[-1] + 5 for t in tensors])])
    out = torch.full((int(starts[-1]) + 1,), float('nan'), device=DEV)
    audio.downmix_into([(t, out, int(a)) for t, a in zip(tensors, starts)])                  # one launch, many items
    got = out.cpu().numpy()
    for t, a in zip(tensors, starts):
        n = t.shape[-1]
        np.testing.assert_array_equal(bits(got[a:a + n]), bits(host_mean(t)), err_msg=f'{tuple(t.shape)} {t.stride()}')
        assert np.isnan(got[a + n:a + n + 5]).all()                                          # nothing written past the end


# --------------------------------------------------------------------------- the session
def stems(seed: int, seconds: float, rate: int, ch: int) -> np.ndarray:
    """[ch, n] float32: one sung line at per-channel gains and noise, with silences for the slicer to cut."""
    rng = np.random.default_rng(seed)
    x = synth.synth_waveform(seed, seconds=seconds, sr=rate, silence_gaps=True).astype(np.float32)
    gains = rng.uniform(0.3, 1.2, (ch, 1)).astype(np.float32)
    return (gains * x[None] + rng.standard_normal((ch, x.shape[0])).astype(np.float32) * np.float32(1e-3)).astype(np.float32)


def same(got, want, frames=False):
    assert got[0] == want[0] and got[1] == want[1]               # offsets and ranges
    assert len(got[2]) == len(want[2])
    for g, w in zip(got[2], want[2]):
        np.testing.assert_array_equal(bits(g['note_midi']), bits(w['note_midi']))
        np.testing.assert_array_equal(g['note_rest'], w['note_rest'])
        np.testing.assert_array_equal(g['note_frames'], w['note_frames'])
    if frames:
        for g, w in zip(got[3], want[3]):
            for a, b in zip(g, w):
                np.testing.assert_array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


@pytest.mark.parametrize('rate', [44100, 48000, 22050])
def test_transcribe_device_equals_sliced_on_the_host_down_mix(sess, rate):
    tensors = []
    for k, ch in enumerate((1, 2, 6, 8, 9)):
        y = stems(100 * k + rate % 97, 9.0 + 2 * k, rate, ch)
        tensors.append((planar, interleaved, wide)[k % 3](y))
    tensors.append(planar(stems(7, 11.0, rate, 1))[0])                                        # [n]
    got = sess.transcribe_device(tensors, [rate] * len(tensors), frames=True)
    for t, g in zip(tensors, got):
        same(g, sess.transcribe_sliced(host_mean(t), rate, frames=True), frames=True)
    # alone, and in another order: results do not depend on the other items
    same(sess.transcribe_device([tensors[3]], [rate])[0], sess.transcribe_sliced(host_mean(tensors[3]), rate))
    for t, g in zip(tensors[::-1], sess.transcribe_device(tensors[::-1], [rate] * len(tensors))):
        same(g, sess.transcribe_sliced(host_mean(t), rate))


def test_reads_wait_for_the_callers_stream_and_end_with_the_call(sess):
    y = stems(11, 12.0, 44100, 2)
    src = planar(y)
    want = sess.transcribe_sliced(host_mean(src), 44100)
    torch.cuda.synchronize()
    side = torch.cuda.Stream(DEV)
    with torch.cuda.stream(side):
        t = torch.zeros_like(src)
        torch.cuda._sleep(200_000_000)                           # the producer is still busy when the call is made
        t.copy_(src)
        got = sess.transcribe_device([t], [44100])[0]            # no synchronise in between
        t.fill_(0.25)                                            # overwritten as soon as the call returns
        again = sess.transcribe_device([t], [44100])[0]
    same(got, want)
    same(again, sess.transcribe_sliced(np.full(y.shape[1], 0.25, np.float32), 44100))


def test_refusals_touch_nothing_and_leave_the_session_usable(sess):
    good = planar(stems(21, 6.0, 44100, 2))
    g = audio.device_audio(good, 0, 't', 44100)
    host = np.zeros((2, 1000), np.float32)

    def item(**kw):
        d = _lib.DeviceAudio.from_buffer_copy(g)
        for k, v in kw.items():
            setattr(d, k, v)
        return d
    cases = [(item(data=None), 'data is NULL'),
             (item(frames=-1), '-1 frames'),
             (item(channels=0), '0 channels'),
             (item(channels=129), '129 channels'),
             (item(frame_stride=2), 'none of the down-mix layouts'),
             (item(data=host.ctypes.data, frames=1000, channel_stride=1000), 'not device memory of device 0 (host memory)'),
             (item(device=torch.cuda.device_count()), 'device'),
             (item(sample_rate=0), 'sample rate 0'),
             (item(frames=1, channel_stride=1, frame_stride=1, sample_rate=48000), 'too small to resample'),
             (item(sample_rate=44_100_000), 'below the table')]       # a rate pair the resampler refuses
    if torch.cuda.device_count() > 1:
        cases.append((item(device=1), 'not device memory of device 1'))
    want = sess.transcribe_sliced(host_mean(good), 44100)
    spare = nsess.Notes()
    for bad, msg in cases:
        held = nsess.Notes()
        sess.transcribe_sliced(host_mean(good)[:44100], 44100, notes=held)
        before = held.results(sess.timestep)
        arr = (_lib.DeviceAudio * 2)(g, bad)
        outs = (C.c_void_p * 2)(spare.handle, held.handle)
        rc = sess.lib.some_session_transcribe_device(sess.handle, arr, 2, None, outs)
        err = sess.lib.some_last_error().decode()
        assert rc != 0 and 'some_session_transcribe_device: item 1: ' in err and msg in err, err
        after = held.results(sess.timestep)
        assert after[0] == before[0] and all(bits(a['note_midi']).tolist() == bits(b['note_midi']).tolist()
                                             for a, b in zip(after[1], before[1]))
        held.close()
        same(sess.transcribe_device([good], [44100])[0], want)          # usable afterwards
    # shared notes, and the wrapper's refusals before any native call
    n = nsess.Notes()
    arr = (_lib.DeviceAudio * 2)(g, g)
    outs = (C.c_void_p * 2)(n.handle, n.handle)
    assert sess.lib.some_session_transcribe_device(sess.handle, arr, 2, None, outs) != 0
    assert 'item 1: shares its some_notes with item 0' in sess.lib.some_last_error().decode()
    for bad, msg in ((good.cpu(), 'item 1: a CUDA tensor expected'), (good.double(), 'item 1: float32'),
                     (good[:, ::2], 'item 1: .*none of the down-mix layouts')):
        with pytest.raises(ValueError, match=msg):
            sess.transcribe_device([good, bad])
    with sess.stream(44100) as st:
        assert st.lib.some_stream_push_device(st.handle, C.byref(item(sample_rate=48000)), st.notes.handle) != 0
        assert 'some_stream_push_device: the audio is at 48000 Hz, the stream at 44100 Hz' in st.lib.some_last_error().decode()
        same(concat([st.push(good), st.finish()]), want)                # the stream is untouched
    with sess.stream_encoded() as st:
        a = audio.device_audio(good, 0, 't', 44100)
        assert st.lib.some_stream_push_device(st.handle, C.byref(a), st.notes.handle) != 0
        assert 'encoded stream' in st.lib.some_last_error().decode()
    same(sess.transcribe_device([good], [44100])[0], want)


# --------------------------------------------------------------------------- threads
def wav16(x, rate):
    import struct
    raw = np.clip(np.round(x * 32768), -32768, 32767).astype('<i2').tobytes()
    fmt = struct.pack('<HHIIHH', 1, 1, rate, rate * 2, 2, 16)
    body = b'WAVE' + b'fmt ' + struct.pack('<I', 16) + fmt + b'data' + struct.pack('<I', len(raw)) + raw
    return b'RIFF' + struct.pack('<I', len(body)) + body


def test_device_calls_from_threads_merge_with_sliced_and_encoded_calls(sess):
    long_items = [wav16(synth.synth_waveform(4242, seconds=600.0, silence_gaps=True) * np.float32(0.8), 44100)] * 2
    dev = [planar(stems(300 + i, 8.0 + i, (44100, 48000)[i % 2], 2)) for i in range(4)]
    host = [synth.synth_waveform(310 + i, seconds=10.0, silence_gaps=True) for i in range(2)]
    enc = [wav16(synth.synth_waveform(320, seconds=7.0, silence_gaps=True), 44100)]
    want_dev = [sess.transcribe_sliced(host_mean(t), (44100, 48000)[i % 2]) for i, t in enumerate(dev)]
    want_host = [sess.transcribe_sliced(x) for x in host]
    want_enc = sess.transcribe_encoded(enc)
    torch.cuda.synchronize()
    out, threads = {}, []

    def start(name, fn):
        def work():
            try:
                out[name] = fn()
            except Exception as e:                              # noqa: BLE001  (checked below)
                out[name] = e
        th = threading.Thread(target=work)
        th.start()
        threads.append(th)

    def wait_for(pred, what):
        end = time.monotonic() + 120
        while not pred(sess.stats()):
            assert time.monotonic() < end, f'timed out waiting for {what}'
            time.sleep(0.0005)
    before = sess.stats()
    start('long', lambda: sess.transcribe_encoded(long_items))
    wait_for(lambda st: st['calls'] == before['calls'] + 1 and st['queued'] == 0, 'the long call')
    calls = [(('dev', i), lambda i=i: sess.transcribe_device([dev[i]], [(44100, 48000)[i % 2]])[0]) for i in range(4)]
    calls += [(('host', i), lambda i=i: sess.transcribe_sliced(host[i])) for i in range(2)] + [('enc', lambda: sess.transcribe_encoded(enc))]
    for q, (name, fn) in enumerate(calls, 1):
        start(name, fn)
        wait_for(lambda st, q=q: st['queued'] == q, f'{name} to queue')
    for th in threads:
        th.join()
    after = sess.stats()
    assert after['steps'] - before['steps'] == 2 and after['max_calls'] >= len(calls)
    for i in range(4):
        same(out[('dev', i)], want_dev[i])
    for i in range(2):
        same(out[('host', i)], want_host[i])
    same(out['enc'][0], want_enc[0])


# --------------------------------------------------------------------------- streams
def concat(results):
    offs, ranges, notes = [], [], []
    for o, r, n in results:
        offs += o
        ranges += r
        notes += n
    return offs, ranges, notes


@pytest.mark.parametrize('rate, make', [(44100, planar), (48000, interleaved), (22050, wide)])
def test_device_pushes_mixed_with_host_pushes_give_the_host_chunks(sess, rate, make):
    y = stems(400 + rate % 89, 40.0, rate, 2)
    t = make(y)
    m = host_mean(t)
    rng = np.random.default_rng(rate)
    cuts = np.sort(rng.choice(np.arange(1, m.shape[0]), size=12, replace=False))
    bounds = list(zip([0, *cuts], [*cuts, m.shape[0]]))
    with sess.stream(rate) as st:
        want = concat([st.push(m[a:b]) for a, b in bounds] + [st.finish()])
    with sess.stream(rate) as st:
        got = concat([st.push(t[:, a:b] if k % 3 else m[a:b]) for k, (a, b) in enumerate(bounds)] + [st.finish()])
    same(got, want)
    same(want, sess.transcribe_sliced(m, rate))


def test_push_device_many_across_rates(sess):
    ys = [stems(500, 30.0, 44100, 2), stems(501, 25.0, 48000, 6)]
    ts = [planar(ys[0]), interleaved(ys[1])]
    rates = [44100, 48000]
    ms = [host_mean(t) for t in ts]
    streams = [sess.stream(r) for r in rates]
    try:
        got = [[], []]
        halves = [(0, 500000), (500000, None)]
        for k, (a, b) in enumerate(halves):
            res = sess.push_device_many([(st, t[:, a:b]) for st, t in zip(streams, ts)], finish=[k == 1, k == 1])
            for i in range(2):
                got[i].append(res[i])
    finally:
        for st in streams:
            st.close()
    for i in range(2):
        same(concat(got[i]), sess.transcribe_sliced(ms[i], rates[i]))


# --------------------------------------------------------------------------- two devices
def test_items_on_a_second_device_and_a_two_device_session(path):
    if torch.cuda.device_count() < 2:
        pytest.skip('two GPUs needed')
    y = stems(600, 14.0, 48000, 2)
    on1 = [torch.from_numpy(y).to('cuda:1'), torch.from_numpy(np.ascontiguousarray(y.T)).to('cuda:1').t()]
    for devices in (0, [0, 1]):
        s = nsess.Session(path, devices)
        try:
            got = s.transcribe_device(on1 + [planar(y)], [48000] * 3)
            for t, g in zip(on1 + [planar(y)], got):
                same(g, s.transcribe_sliced(host_mean(t), 48000))
        finally:
            s.close()


# --------------------------------------------------------------------------- the Python host
def test_transcribe_recordings_takes_cuda_tensors(ckpt):
    ins = plugin.MIDIExtractionInference(config=synth.named_config('two_head'), model_path=ckpt, device='cuda:0')
    rates = [44100, 48000, 44100, 22050]
    tensors = [planar(stems(700, 12.0, 44100, 2)), interleaved(stems(701, 9.0, 48000, 9)),
               wide(stems(702, 5.0, 44100, 6)), planar(stems(703, 7.0, 22050, 1))[0]]
    hosts = [host_mean(t) for t in tensors]
    got = batch.transcribe_recordings(ins, tensors, rates=rates)
    want = batch.transcribe_recordings(ins, hosts, rates=rates)
    mixed = batch.transcribe_recordings(ins, [tensors[0], hosts[1], tensors[2], hosts[3]], rates=rates)
    for res in (got, mixed):
        assert len(res) == len(want)
        for (go, gn), (wo, wn) in zip(res, want):
            assert go == wo and len(gn) == len(wn)
            for a, b in zip(gn, wn):
                np.testing.assert_array_equal(bits(a['note_midi']), bits(b['note_midi']))
                np.testing.assert_array_equal(a['note_rest'], b['note_rest'])
                np.testing.assert_array_equal(a['note_dur'], b['note_dur'])
