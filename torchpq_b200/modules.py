"""Module plumbing shared by the index and its codecs.

Checkpoint compatibility with the reference: its objects are ``nn.Module``s whose state is
a set of registered buffers, and its ``load_state_dict`` drops and re-registers every
top-level buffer so shapes may change between save and load
(torchpq/CustomModule.py:14-23; README.md:90-97).  ``StateModule`` keeps that contract and
the same buffer names, so a ``state_dict`` saved by ``torchpq.index.IVFPQIndex`` loads here.
"""
from __future__ import annotations

import functools
import math

import torch
import torch.nn as nn


class StateModule(nn.Module):
    verbose = 0

    def print_message(self, text, min_verbosity=0):
        if self.verbose >= min_verbosity:
            print(f"{type(self).__name__}: {text}")

    def load_state_dict(self, state_dict, strict=True):  # noqa: D401 - reference semantics, see module docstring
        for key, value in state_dict.items():
            if "." in key:
                continue
            assert hasattr(self, key), f"attribute {key} does not exist"
            delattr(self, key)
            self.register_buffer(key, value)
        for name, child in self.named_children():
            prefix = name + "."
            child.load_state_dict({k[len(prefix):]: v for k, v in state_dict.items() if k.startswith(prefix)})
        self._state_changed()

    def _state_changed(self):
        pass


def on_device(device_of):
    """Decorator: run the function with the CUDA device of its data made current, ``device_of(*args, **kwargs)``.
    The library launches every kernel on the current device, into the stream it is given, and reads the current
    device's SM count; a stream of another device makes the launch fail.  So an index on cuda:1 works while cuda:0
    is current.  Data already on the current device, or not on a CUDA device at all (the function's own checks reject
    it), runs as is."""
    def wrap(fn):
        @functools.wraps(fn)
        def run(*args, **kwargs):
            dev = device_of(*args, **kwargs)
            if dev.type != "cuda" or dev.index is None or dev.index == torch.cuda.current_device():
                return fn(*args, **kwargs)
            with torch.cuda.device(dev):
                return fn(*args, **kwargs)
        return run
    return wrap


on_index_device = on_device(lambda self, *a, **k: self._address2id.device)   # a method of an index
on_data_device = on_device(lambda x, *a, **k: x.device)                      # a function of a tensor


def _fingerprint(*tensors):
    return tuple((t.data_ptr(), t._version, tuple(t.shape)) if t is not None else None for t in tensors)


class StreamCache:
    """A device-side cache (a norm table, a scan layout) filled by kernels on the stream current at construction, and
    read from any stream.  Construct it after the cache's last kernel: it records an event there, and ``get`` makes a
    reader on another stream wait on that event, so a search never reads a half-built cache.  The wait is skipped while
    the reader's stream is capturing a CUDA graph: ``torch.cuda.graph`` synchronises the device before it captures, so
    the cache is complete by then, and a capture may not wait on an event recorded outside it."""

    def __init__(self, value, device):
        # built inside a capture, the cache would live in the graph's pool and be filled only on replay, and eager
        # searches would then read it unfilled
        assert not torch.cuda.is_current_stream_capturing(), \
            "a cache was built inside a CUDA graph capture: run the call once eagerly before capturing it"
        self.value = value
        self._stream = torch.cuda.current_stream(device)
        self._ready = torch.cuda.Event()
        self._ready.record(self._stream)

    def get(self):
        cur = torch.cuda.current_stream(self._stream.device)
        if cur.cuda_stream != self._stream.cuda_stream and not torch.cuda.is_current_stream_capturing():
            cur.wait_event(self._ready)
        return self.value


class IdContainer(StateModule):
    """The id bookkeeping of BaseContainer (container/BaseContainer.py:30-110) that IVFPQIndex and FlatIndex share: the
    ``_address2id`` / ``_id2address`` buffers, ``capacity``, ``max_id`` (tracked, and re-derived from ``_address2id``
    after a checkpoint load, where the reference restarts it at -1) and the two lookups.  The inverse map is rebuilt
    lazily, whenever ``_address2id`` has changed since it was built: its fingerprint (pointer, ``_version``, shape) sees
    every write through torch, and a writer that bypasses ``_version`` (a kernel writing through the raw pointer,
    build.container_add) calls ``_ids_changed``.  Subclasses register both buffers and set ``_max_id = -1`` and
    ``_id2address_fp = None``."""

    def _ids_changed(self):
        """``_address2id`` was written where its ``_version`` does not see it: drop the inverse map."""
        self._id2address_fp = None

    @property
    def capacity(self):
        return self._address2id.shape[0]

    @property
    def max_id(self):
        return self._max_id

    def _refresh_max_id(self):
        a2i = self._address2id
        self._max_id = int(a2i.max().item()) if a2i is not None and a2i.numel() else -1
        self._ids_changed()

    def get_id_by_address(self, address):
        """BaseContainer.get_id_by_address (BaseContainer.py:58-65) -- plain tensor indexing, not on the hot path."""
        assert address.dtype == torch.int64
        mask = (0 <= address) & (address < self.capacity)
        ids = torch.ones_like(address) * -1
        ids[mask] = self._address2id[address[mask]]
        return ids

    def get_address_by_id(self, ids):
        """BaseContainer.get_address_by_id with the inverse id map (BaseContainer.py:78-110; both indexes build their
        container with use_inverse_id_mapping=True, IVFPQIndex.py:39, FlatIndex.py:27)."""
        assert ids.dtype == torch.int64
        ids = ids.to(self._address2id.device)
        if self._id2address is None or self._id2address_fp != _fingerprint(self._address2id):
            a2i_v, a2i_i = self._address2id.sort()
            keep = a2i_v >= 0
            if a2i_v.numel():                                          # never trust a stale _max_id (checkpoint loads)
                self._max_id = max(self._max_id, int(a2i_v[-1].item()))
            id2a = -torch.ones(self._max_id + 1, dtype=torch.long, device=ids.device)
            id2a[a2i_v[keep]] = a2i_i[keep]
            delattr(self, "_id2address")
            self.register_buffer("_id2address", id2a)
            self._id2address_fp = _fingerprint(self._address2id)
        # bounded by the map's own length too: a lookup can never index past it, even were the map stale
        mask = (0 <= ids) & (ids <= self._max_id) & (ids < self._id2address.shape[0])
        address = torch.ones_like(ids) * -1
        address[mask] = self._id2address[ids[mask]]
        return address


def live_prefix(address2id):
    """The number of live slots (address2id >= 0) of a store whose live slots must be the prefix [0, n_items), as
    FlatIndex and RefineFlatIndex keep it; a checkpoint whose live slots are not a prefix is refused."""
    live = address2id >= 0
    n = int(live.sum().item())
    assert bool(live[:n].all().item()), "the live slots of a flat index must be the prefix [0, n_items)"
    return n


def prefix_remove(address2id, address, n_items):
    """FlatContainer.remove's rule (FlatContainer.py:160-190) for a store whose live slots are the prefix [0, n_items):
    the surviving items of the last n_removed slots move, in ascending order, into the removed slots below them.
    Addresses outside the live prefix are ignored.  Updates address2id in place and returns (n_removed, dst, src, tail):
    the caller moves its rows src -> dst and clears the slots of `tail` (a slice)."""
    address = address[(0 <= address) & (address < n_items)].unique(sorted=True)
    n_removed = address.shape[0]
    if n_removed == 0:
        return 0, None, None, None
    tail = slice(n_items - n_removed, n_items)
    address2id[address] = -1
    keep = address2id[tail] != -1                                    # surviving items of the tail, ascending
    n_move = int(keep.sum().item())
    dst = address[:n_move]                                           # the removed slots below the tail
    src = torch.arange(n_items - n_removed, n_items, dtype=torch.long, device=address2id.device)[keep]
    address2id[dst] = address2id[src].clone()
    address2id[tail] = -1
    return n_removed, dst, src, tail


def k1_of(k, k_factor):
    """The first pass's depth of a re-ranked search (IVFPQRIndex, RefineFlatIndex): k1 = min(1024, max(k,
    ceil(k_factor * k))) candidates, re-scored exactly and cut to k."""
    return min(1024, max(k, math.ceil(k_factor * k)))


class _Centroids(StateModule):
    """Stands where the reference has KMeans / MultiKMeans: owner of the ``centroids`` buffer
    (clustering/KMeans.py:74, clustering/MultiKMeans.py:73)."""

    def __init__(self):
        super().__init__()
        self.register_buffer("centroids", None)


class Codec(StateModule):
    """BaseCodec (codec/BaseCodec.py:5-17): ``_is_trained`` flag + a ``kmeans.centroids`` codebook."""

    def __init__(self):
        super().__init__()
        self.register_buffer("_is_trained", torch.tensor(False))
        self.kmeans = _Centroids()

    @property
    def is_trained(self) -> bool:
        # cached as a Python bool: `.item()` on a CUDA `_is_trained` would be a host sync on every search
        t = self._is_trained
        key = (t.data_ptr(), t._version)
        if getattr(self, "_trained_key", None) != key:
            self._trained_cache, self._trained_key = bool(t.item()), key
        return self._trained_cache

    @property
    def codebook(self):
        return self.kmeans.centroids if self.is_trained else None

    def set_codebook(self, centroids: torch.Tensor):
        self.kmeans.register_buffer("centroids", centroids)
        self._is_trained.data = torch.tensor(True)
