"""Multi-GPU data parallelism for the SOME inference path (new: the reference has none —
inference/base_infer.py:46-53 is a serial single-device loop).

Clips are independent units, so the path shards with NO data-path collective: every rank (one process
per GPU) runs mel -> trunk -> decode on its own clips.  The only exchange is ONE all-gather of the packed
per-clip note records (a few KB..MB) so that every rank ends with the full, input-ordered result list.

* ``shard_clips``: longest-processing-time greedy assignment with cost T * (dense + c * T) so the quadratic
  attention term of long clips is balanced.
* ``gather_results``: fixed-size uint8 slab per rank [counts i32 | dur i32 | midi f32 | rest u8] -> one
  ``all_gather_into_tensor`` (NCCL over NVLink on GPUs, gloo in the CPU tests) -> unpack in input order.
"""
from __future__ import annotations

import collections.abc
import functools
from typing import Dict, List, Sequence

import numpy as np
import torch
import torch.distributed as dist

from .session import shard_clips as shard_owner

HOP = 512
# per-frame cost model (SURVEY.md §8d): 103.31 MFLOP dense + 2 * 8 blocks * 2 * T * 512 FLOP attention
_DENSE, _ATT = 103.31e6, 16384.0


def clip_cost(num_samples: int) -> float:
    t = 1 + num_samples // HOP
    return t * (_DENSE + _ATT * t)


@functools.lru_cache(maxsize=64)
def _shard_clips(lengths: tuple, world: int):
    # LPT over clip_cost, in order of (-cost, index), each clip to the least loaded rank (ties: the lowest): some_shard_clips,
    # the rule a multi-device native session assigns its chunks by
    shards: List[List[int]] = [[] for _ in range(world)]
    for i, r in enumerate(shard_owner(lengths, world)):
        shards[r].append(i)
    return tuple(tuple(s) for s in shards)


def shard_clips(lengths: Sequence[int], world: int) -> List[List[int]]:
    """Deterministic LPT assignment: returns, per rank, the (ascending) global indices of its clips.  Memoised on the
    lengths: a serving loop shards the same batch shape step after step, and at 8 ranks x 64 clips the pure-Python assignment
    is milliseconds -- more than the collective it prepares."""
    return [list(s) for s in _shard_clips(tuple(int(n) for n in lengths), int(world))]


def _slab_layout(lengths: Sequence[int], shard: Sequence[int]):
    frames = [1 + lengths[i] // HOP for i in shard]
    b, m = len(shard), int(sum(frames))
    return b, m, frames


def slab_bytes(lengths: Sequence[int], shards: Sequence[Sequence[int]]) -> int:
    worst = 0
    for s in shards:
        b, m, _ = _slab_layout(lengths, s)
        worst = max(worst, 4 * b + 9 * m)
    return (worst + 15) & ~15


def pack_results(results: List[Dict[str, np.ndarray]], frames: Sequence[int], nbytes: int, timestep: float) -> np.ndarray:
    """[counts i32 [b] | dur i32 [m] | midi f32 [m] | rest u8 [m]], notes of clip j at offset cu[j]."""
    b, m = len(results), int(sum(frames))
    slab = np.zeros(nbytes, dtype=np.uint8)
    counts = slab[:4 * b].view(np.int32)
    dur = slab[4 * b:4 * b + 4 * m].view(np.int32)
    midi = slab[4 * b + 4 * m:4 * b + 8 * m].view(np.float32)
    rest = slab[4 * b + 8 * m:4 * b + 9 * m]
    r0 = 0
    for j, (res, t) in enumerate(zip(results, frames)):
        n = len(res['note_midi'])
        counts[j] = n
        dur[r0:r0 + n] = np.rint(res['note_dur'] / timestep).astype(np.int32)
        midi[r0:r0 + n] = res['note_midi']
        rest[r0:r0 + n] = res['note_rest']
        r0 += t
    return slab


def unpack_results(slab: np.ndarray, frames: Sequence[int], timestep: float) -> List[Dict[str, np.ndarray]]:
    b, m = len(frames), int(sum(frames))
    counts = slab[:4 * b].view(np.int32)
    dur = slab[4 * b:4 * b + 4 * m].view(np.int32)
    midi = slab[4 * b + 4 * m:4 * b + 8 * m].view(np.float32)
    rest = slab[4 * b + 8 * m:4 * b + 9 * m]
    out, r0 = [], 0
    for j, t in enumerate(frames):
        n = int(counts[j])
        out.append({'note_midi': midi[r0:r0 + n].copy(),
                    'note_dur': dur[r0:r0 + n].astype(np.int64) * timestep,
                    'note_rest': rest[r0:r0 + n].astype(bool)})
        r0 += t
    return out


def gather_results(local: List[Dict[str, np.ndarray]], lengths: Sequence[int], shards: Sequence[Sequence[int]],
                   timestep: float, device=None, group=None) -> List[Dict[str, np.ndarray]]:
    """One all-gather of the packed note records; returns the results of ALL clips in input order."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    nbytes = slab_bytes(lengths, shards)
    _, _, my_frames = _slab_layout(lengths, shards[rank])
    mine = torch.from_numpy(pack_results(local, my_frames, nbytes, timestep))
    if device is not None:
        mine = mine.to(device, non_blocking=True)
    everything = torch.empty(world * nbytes, dtype=torch.uint8, device=mine.device)
    dist.all_gather_into_tensor(everything, mine, group=group)
    host = everything.cpu().numpy()
    merged: List[Dict[str, np.ndarray]] = [None] * len(lengths)  # type: ignore
    for r in range(world):
        _, _, frames = _slab_layout(lengths, shards[r])
        for idx, res in zip(shards[r], unpack_results(host[r * nbytes:(r + 1) * nbytes], frames, timestep)):
            merged[idx] = res
    return merged


class ShardedResults(collections.abc.Sequence):
    """The ordered result list of a data-parallel infer: behaves like the ``List[Dict]`` of ``BaseInference.infer`` but
    unpacks a rank's slab only when one of ITS clips is first touched — a caller that consumes only its own shard (or rank 0
    writing the output files) never pays for converting world x clips note records on every rank."""

    def __init__(self, n: int, owner: Sequence[int], unpackers):
        self._items: List = [None] * n
        self._owner = list(owner)              # clip index -> rank
        self._unpackers = list(unpackers)      # rank -> callable() -> [(clip index, result dict), ...] or None once done

    def _materialise_rank(self, r: int):
        fn = self._unpackers[r]
        if fn is not None:
            self._unpackers[r] = None
            for idx, res in fn():
                self._items[idx] = res

    def materialise(self) -> List[Dict[str, np.ndarray]]:
        for r in range(len(self._unpackers)):
            self._materialise_rank(r)
        return self._items

    def __len__(self):
        return len(self._items)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(len(self)))]
        if i < 0:
            i += len(self._items)
        if self._items[i] is None and self._owner[i] >= 0:
            self._materialise_rank(self._owner[i])
        return self._items[i]


def infer_sharded(plugin, waveforms: Sequence[np.ndarray], group=None) -> List[Dict[str, np.ndarray]]:
    """Data-parallel ``infer``: every rank holds the same ``waveforms`` list (or at least its own shard's
    entries), processes its shard and all ranks return the full ordered result list.

    With the CUDA engine and NCCL the decode kernel's packed note slab never takes a detour through Python: each rank
    enqueues its shard, the device slabs are all-gathered (one ``all_gather_into_tensor`` over NVLink), and the gathered
    buffer is copied to the host once and unpacked with the layouts every rank can derive from the clip lengths."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    lengths = [int(w.shape[0]) for w in waveforms]
    shards = shard_clips(lengths, world)
    eng = getattr(plugin, 'model', None)
    if dist.get_backend(group) == 'nccl' and hasattr(eng, 'enqueue'):
        import threading
        import weakref
        layouts = [eng.slab_layout_cached([lengths[i] for i in s]) if s else (np.zeros(1, np.int32), [], 0) for s in shards]
        nbytes = max(16, max(l[2] for l in layouts))
        with getattr(plugin, '_lock', threading.Lock()), torch.cuda.device(eng.device):
            # The previous call's results unpack lazily out of the page-locked landing buffer this call is about to overwrite:
            # whatever the caller has not touched yet is unpacked now (normally nothing: no copy of the gathered bytes is made).
            prev = getattr(eng, '_lazy_results', None)
            prev = prev() if prev is not None else None
            if prev is not None:
                prev.materialise()
            mine = [waveforms[i] for i in shards[rank]]
            # persistent gather buffer (device) + page-locked landing buffer (host); the decode kernel writes this rank's
            # notes STRAIGHT into its slot of the gather buffer and the collective runs in place (send = own slot)
            buf = getattr(eng, '_gather', None)
            if buf is None or buf[0].numel() < world * nbytes:
                buf = (torch.empty(world * nbytes, dtype=torch.uint8, device=eng.device),
                       torch.empty(world * nbytes, dtype=torch.uint8).pin_memory())
                eng._gather = buf
            gathered, landing = buf[0][:world * nbytes], buf[1][:world * nbytes]
            slot = gathered[rank * nbytes:(rank + 1) * nbytes]
            if mine:
                eng.enqueue(mine, quantized=getattr(plugin, 'quantized', False), out=slot)
            dist.all_gather_into_tensor(gathered, slot, group=group)
            landing.copy_(gathered, non_blocking=True)
            torch.cuda.current_stream(eng.device).synchronize()
            host = landing.numpy()             # no copy: unpacking gathers the used rows out of it (Engine.unpack)

        def unpacker(r):
            cu_r, layout_r, _ = layouts[r]
            return lambda: list(zip(shards[r], eng.unpack_slab(host[r * nbytes:(r + 1) * nbytes], cu_r, layout_r)))

        owner = [-1] * len(lengths)
        for r, s in enumerate(shards):
            for i in s:
                owner[i] = r
        out = ShardedResults(len(lengths), owner, [unpacker(r) if layouts[r][1] else None for r in range(world)])
        out._materialise_rank(rank)            # this rank's own clips eagerly, the others on first touch
        eng._lazy_results = weakref.ref(out)
        return out
    local = plugin.infer([waveforms[i] for i in shards[rank]])
    dev = getattr(eng, 'device', None) if dist.get_backend(group) == 'nccl' else None
    return gather_results(local, lengths, shards, plugin.timestep, device=dev, group=group)


def infer_sliced_sharded(plugin, waveform: np.ndarray, slicer, group=None):
    """C5 across GPUs (SURVEY.md §8d): ONE long recording -> slicer -> the chunks sharded over the ranks -> all ranks return
    (chunk offsets in seconds, notes of every chunk in order).

    Every rank holds the recording and cuts it itself (the device RMS + host slicer cost well under a millisecond of GPU
    time and are deterministic, so no broadcast of the cut list is needed); the chunks are zero-copy views, each rank stages
    and uploads only its own shard, and the exchange is the same single all-gather of packed notes as ``infer_sharded``."""
    ranges = slicer.ranges(waveform)
    chunks = [waveform[..., a:b] for a, b in ranges]
    notes = infer_sharded(plugin, chunks, group=group) if chunks else []
    return [a / slicer.sr for a, _ in ranges], notes
