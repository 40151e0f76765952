"""ctypes binding of libkueue_b200.so — the same C-ABI a cgo shim binds
(include/kueue_b200.h, INTEGRATION.md).  There is NO CPU fallback: if the CUDA
library is missing or no device is present, construction raises."""
from __future__ import annotations

import ctypes as C
import os
import weakref

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KUEUE_B200_LIB") or os.path.join(_HERE, "libkueue_b200.so")  # override: instrumented builds
_LIB = None

EXPORTS = ["kb_create", "kb_destroy", "kb_last_error", "kb_alloc_pinned", "kb_free_pinned", "kb_version",
           "kb_tree_eval", "kb_run_cycle", "kb_run_drain", "kb_tas_find", "kb_upload", "kb_cycle_resident", "kb_download", "kb_get_stats", "kb_set_profile",
           "kb_alloc_cycle_out"]


class KueueB200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libkueue_b200 error {code}: {msg}")
        self.code = code


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(LIB_PATH)
        L.kb_last_error.restype = C.c_char_p
        L.kb_last_error.argtypes = [C.c_void_p]
        for name in EXPORTS:
            if name not in ("kb_last_error", "kb_destroy"):
                getattr(L, name).restype = C.c_int32
        L.kb_destroy.restype = None
        L.kb_destroy.argtypes = [C.c_void_p]
        _LIB = L
    return _LIB


def pinned_array(shape, dtype) -> "np.ndarray":
    """numpy view over page-locked host memory from kb_alloc_pinned (what the Go shim
    uses for its SoA buffers so the GC never moves them and H2D copies are DMA)."""
    import numpy as np
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) if shape != () else 1
    ptr = C.c_void_p()
    rc = lib().kb_alloc_pinned(C.byref(ptr), C.c_uint64(max(1, n * dtype.itemsize)))
    if rc != 0:
        raise KueueB200Error(rc, "kb_alloc_pinned failed")
    buf = (C.c_char * max(1, n * dtype.itemsize)).from_address(ptr.value)
    weakref.finalize(buf, _free_pinned, ptr.value)  # released when the last numpy view of the block is gone
    arr = np.frombuffer(buf, dtype=dtype, count=n).reshape(shape)
    return arr


def _free_pinned(address: int) -> None:
    try:
        lib().kb_free_pinned(C.c_void_p(address))
    except Exception:  # noqa: BLE001 — interpreter shutdown
        pass


def pin_snapshot(snap: abi.FlatSnapshot) -> abi.FlatSnapshot:
    """Copy of `snap` whose arrays live in ONE block of pinned host memory (256 B aligned sub-arrays, the static
    tables first).  The library recognises per-cycle tables that sit close together in host memory and moves them
    with a single DMA (span upload, kb_api.cu) — the layout the Go shim gets by carving its SoA buffers out of one
    kb_alloc_pinned block."""
    import numpy as np
    out = abi.FlatSnapshot(n_cq=snap.n_cq, n_cohort=snap.n_cohort, n_flavor=snap.n_flavor, n_resource=snap.n_resource,
                           pods_resource=snap.pods_resource, flags=snap.flags, now_ns=snap.now_ns)
    static = [k for k in snap.arrays if k in abi.STATIC_FIELDS]
    order = static + [k for k in snap.arrays if k not in abi.STATIC_FIELDS]
    pad = lambda n: (max(1, n) + 255) & ~255  # noqa: E731
    total = sum(pad(snap.arrays[k].nbytes) for k in order)
    block = pinned_array((total,), np.uint8)
    off = 0
    for k in order:
        v = snap.arrays[k]
        a = block[off:off + v.nbytes].view(v.dtype).reshape(v.shape)
        a[...] = v
        out.arrays[k] = a
        off += pad(v.nbytes)
    out._pinned_block = block
    out.static_generation = snap.static_generation
    out.afs_alpha = snap.afs_alpha
    out.afs_half_life_ns, out.afs_sampling_ns = snap.afs_half_life_ns, snap.afs_sampling_ns
    return out


def pin_cycle_out(out: abi.CycleOut) -> abi.CycleOut:
    """Re-point the output buffers at ONE page-locked block from kb_alloc_cycle_out (laid out like the library's
    device-side result tables, so the eight per-entry / per-podset tables come back with a single DMA)."""
    import numpy as np
    H, (P, R) = out.decision.shape[0], out.ps_flavor.shape
    cells = 0 if out.node_usage is None else int(out.node_usage.size)
    s = abi.kb_cycle_out()
    rc = lib().kb_alloc_cycle_out(C.c_int32(H), C.c_int32(P), C.c_int32(R), C.c_int32(out.struct.tgt_capacity), C.c_int64(cells), C.byref(s))
    if rc != 0:
        raise KueueB200Error(rc, "kb_alloc_cycle_out failed")

    def view(ptr, like):
        n = max(1, like.size * like.dtype.itemsize)
        buf = (C.c_char * n).from_address(C.cast(ptr, C.c_void_p).value)
        a = np.frombuffer(buf, dtype=like.dtype, count=like.size).reshape(like.shape)
        a[...] = like
        return a
    for name in ("decision", "mode", "borrow", "commit_rank", "ps_flavor", "ps_res_mode", "ps_tried_idx", "ps_count",
                 "tgt_start", "tgt_adm", "tgt_reason", "node_usage"):
        old = getattr(out, name)
        if old is None:
            continue
        setattr(out, name, view(getattr(s, name), old))
    out.struct = s
    # the block lives as long as the CycleOut object (its arrays are views into it)
    weakref.finalize(out, _free_pinned, C.cast(s.decision, C.c_void_p).value)
    return out


class Evaluator:
    """One kb_handle (one CUDA device, one stream)."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        cfg = abi.kb_config(device, 0)
        rc = lib().kb_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            raise KueueB200Error(rc, lib().kb_last_error(None).decode())

    def close(self):
        if self._h:
            lib().kb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise KueueB200Error(rc, lib().kb_last_error(self._h).decode())

    def tree_eval(self, snap: abi.FlatSnapshot) -> abi.TreeOut:
        out = abi.TreeOut(snap)
        s = snap.as_struct()
        self._check(lib().kb_tree_eval(self._h, C.byref(s), C.byref(out.struct)))
        return out

    def run_cycle(self, snap: abi.FlatSnapshot, out: abi.CycleOut | None = None) -> abi.CycleOut:
        out = out or abi.CycleOut(snap)
        s = snap.as_struct(cached=True)
        self._check(lib().kb_run_cycle(self._h, C.byref(s), C.byref(out.struct)))
        out.n_targets = out.struct.n_targets
        return out

    def run_drain(self, snap: abi.FlatSnapshot, out: "abi.DrainOut | None" = None, max_cycles: int = 10_000) -> "abi.DrainOut":
        """kb_run_drain: iterated cycles over whole queues with the queue layer on the device."""
        out = out or abi.DrainOut(snap, max_cycles)
        s = snap.as_struct()
        self._check(lib().kb_run_drain(self._h, C.byref(s), C.byref(out.struct)))
        return out

    def tas_find(self, topo, reqs, capacity: int | None = None):
        """kb_tas_find: topology-aware placement of a batch of podset requests (kueue_b200.tas objects)."""
        from . import tas
        out = tas.TasOut(reqs, capacity if capacity is not None else max(16, int(reqs.count.sum()) + 16))
        self._check(lib().kb_tas_find(self._h, C.byref(topo.struct), C.byref(reqs.struct), C.byref(out.struct)))
        return out

    def upload(self, snap: abi.FlatSnapshot):
        s = snap.as_struct()
        self._check(lib().kb_upload(self._h, C.byref(s)))

    def cycle_resident(self):
        self._check(lib().kb_cycle_resident(self._h))

    def download(self, snap: abi.FlatSnapshot, out: abi.CycleOut | None = None) -> abi.CycleOut:
        out = out or abi.CycleOut(snap)
        self._check(lib().kb_download(self._h, C.byref(out.struct)))
        out.n_targets = out.struct.n_targets
        return out

    def set_profile(self, on: bool):
        self._check(lib().kb_set_profile(self._h, 1 if on else 0))

    def stats(self) -> abi.kb_stats:
        st = abi.kb_stats()
        self._check(lib().kb_get_stats(self._h, C.byref(st)))
        return st
