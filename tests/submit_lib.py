"""b200_pairs_submit for the tests (TEST INFRASTRUCTURE).

Arena         one buffer of every memory kind a submit pass takes slices from, set up before the service starts
submit()      one b200_pairs_submit pass over ctypes
SubmitEngine  tests/trace.run_trace adapter: every op one pass (the endpoint's path with the service running)
"""
import ctypes as C

import numpy as np

from gpu_engine import GpuEngine


class Arena:
    """One buffer of every memory kind b200_pairs_submit takes slices from, carved by a bump allocator:
    plain numpy memory (unregistered: staged in the pinned bounce), b200_mem_alloc_host, page-aligned anonymous
    memory passed to b200_mem_register_host, and device memory.  Allocate it before b200_service_start and free it
    after b200_service_stop: cudaHostRegister / Unregister and frees stay out of the resident kernels' way.
    `nbytes`: one size for every kind, or a dict kind -> size."""
    KINDS = ("plain", "host", "registered", "device")

    def __init__(self, pkg, nbytes):
        import mmap
        self.pkg, L = pkg, pkg.lib()
        self.L = L
        size = nbytes if isinstance(nbytes, dict) else dict.fromkeys(self.KINDS, nbytes)
        self.size = {k: max(int(size.get(k, 1 << 20)), 1 << 20) for k in self.KINDS}
        self._plain = np.zeros(self.size["plain"], np.uint8)
        self._mm = mmap.mmap(-1, self.size["registered"])
        self._reg = np.frombuffer(self._mm, np.uint8)
        self.base = {"plain": self._plain.ctypes.data, "registered": self._reg.ctypes.data,
                     "host": L.b200_mem_alloc_host(self.size["host"]),
                     "device": L.b200_mem_alloc_device(self.size["device"])}
        assert self.base["host"] and self.base["device"], pkg.last_error()
        assert L.b200_mem_register_host(self.base["registered"], self.size["registered"]) == 0, pkg.last_error()
        self.window = {k: (0, self.size[k]) for k in self.KINDS}
        self.reset()

    def part(self, i, k):
        """the i-th of k disjoint windows (one per thread)"""
        import copy
        a = copy.copy(self)
        a.window = {kind: (self.size[kind] // k * i, self.size[kind] // k * (i + 1)) for kind in self.KINDS}
        a.reset()
        return a

    def reset(self):
        self.off = {k: self.window[k][0] for k in self.KINDS}

    def alloc(self, kind, n, mis=0):
        o = (self.off[kind] + 64) // 64 * 64 + mis  # never adjacent to the previous allocation
        assert o + n <= self.window[kind][1], "arena: %s window full" % kind
        self.off[kind] = o + n
        return self.base[kind] + o

    def put(self, kind, ptr, arr):
        if arr.size == 0:
            return
        if kind == "device":
            assert self.L.b200_memcpy(ptr, arr.ctypes.data, arr.size, 0, None) == 0
            assert self.L.b200_stream_sync(None) == 0
        else:
            C.memmove(ptr, arr.ctypes.data, arr.size)

    def get(self, kind, ptr, n):
        out = np.zeros(max(n, 1), dtype=np.uint8)
        if n and kind == "device":
            assert self.L.b200_memcpy(out.ctypes.data, ptr, n, 1, None) == 0
            assert self.L.b200_stream_sync(None) == 0
        elif n:
            C.memmove(out.ctypes.data, ptr, n)
        return out[:n]

    def place(self, bufs, kinds, mis=0):
        """copy `bufs` into the arena, slice i in memory kind kinds[i], with odd gaps between the slices (no two
        adjacent, every alignment mod 16); returns the b200_slice array"""
        sl = []
        for i, (b, kind) in enumerate(zip(bufs, kinds)):
            ptr = self.alloc(kind, b.size, (mis + 5 * i) % 16)
            sl.append((ptr, b.size))
        by_kind = {}
        for (ptr, _), b, kind in zip(sl, bufs, kinds):
            by_kind.setdefault(kind, []).append((ptr, b))
        for kind, items in by_kind.items():
            if kind == "device" and len(items) > 1:  # one upload per kind: the slices' span with the gaps
                lo = min(p for p, _ in items)
                hi = max(p + b.size for p, b in items)
                flat = np.zeros(hi - lo, np.uint8)
                for p, b in items:
                    flat[p - lo:p - lo + b.size] = b
                self.put(kind, lo, flat)
            else:
                for p, b in items:
                    self.put(kind, p, b)
        return self.pkg.make_slices(sl)

    def free(self):
        self.L.b200_mem_unregister_host(self.base["registered"])
        self.L.b200_mem_free_host(self.base["host"])
        self.L.b200_mem_free_device(self.base["device"])


SLICE_AREA = 1024  # kSvcSliceArea: an until-blocked submit op dereferences at most SLICE_AREA - 1 slices


def submit(pkg, sends=(), recvs=(), flags=1):
    """one b200_pairs_submit pass.  sends: (pair handle, slice array, nslices, byte_idx); recvs: (pair handle, dst,
    cap).  Returns (rc, accepted, delivered)."""
    L = pkg.lib()
    so = (pkg.SendOp * max(1, len(sends)))()
    ro = (pkg.RecvOp * max(1, len(recvs)))()
    for i, (h, sl, n, bidx) in enumerate(sends):
        so[i].pair, so[i].slices, so[i].nslices, so[i].byte_idx = h, sl, n, bidx
    for i, (h, dst, cap) in enumerate(recvs):
        ro[i].pair, ro[i].dst, ro[i].cap = h, dst, cap
    acc = (C.c_uint64 * max(1, len(sends)))()
    dlv = (C.c_uint64 * max(1, len(recvs)))()
    rc = L.b200_pairs_submit(so, len(sends), acc, ro, len(recvs), dlv, flags)
    return rc, list(acc)[:len(sends)], list(dlv)[:len(recvs)]


class SubmitEngine(GpuEngine):
    """The endpoint's data path for tests/trace.run_trace: every op is one b200_pairs_submit pass with that one op
    (the service must run).  send / recv: B200_BATCH_ONE_CALL; send_all / recv_drain: B200_BATCH_UNTIL_BLOCKED, and
    like the endpoint a send_all re-submits from the returned position when an op ended at the slice window.
    Slices rotate through the memory kinds of `arena` (and a mix of them) from op to op, destinations through the
    GPU-addressable ones.  The pass does not return `calls`: it is -1 (compare records without it)."""
    SRC = Arena.KINDS + ("mixed",)
    DST = ("host", "registered", "device")

    def __init__(self, pkg, arena, coalesce=False, stamped=False):
        super().__init__(pkg)
        self.arena, self.coalesce, self.stamped = arena, coalesce, stamped
        self.k = 0

    def pair_pair(self, cap, max_sge=30):
        self.pkg.config_set("B200_SEND_COALESCE", int(self.coalesce))
        self.pkg.config_set("B200_RING_STAMPED", int(self.stamped))
        try:
            tx, rx = super().pair_pair(cap, max_sge)
        finally:
            self.pkg.config_set("B200_SEND_COALESCE", 0)
            self.pkg.config_set("B200_RING_STAMPED", 0)
        assert tx.stamped() == self.stamped
        return tx, rx

    def _send(self, p, bufs, byte_idx, flags):
        self.k += 1
        a = self.arena
        a.reset()
        kind = self.SRC[self.k % len(self.SRC)]
        kinds = [Arena.KINDS[(self.k + i) % 4] for i in range(len(bufs))] if kind == "mixed" else [kind] * len(bufs)
        sl = a.place(bufs, kinds, self.k)
        rc, acc, _ = submit(self.pkg, [(p.h, sl, len(bufs), byte_idx)], flags=flags)
        assert rc == 0, self.pkg.last_error()
        return acc[0]

    def _recv(self, p, cap, flags):
        self.k += 1
        a = self.arena
        a.reset()
        kind = self.DST[self.k % len(self.DST)]
        dst = a.alloc(kind, cap, self.k % 16)
        rc, _, dlv = submit(self.pkg, recvs=[(p.h, dst, cap)], flags=flags)
        assert rc == 0, self.pkg.last_error()
        return a.get(kind, dst, dlv[0]).copy()

    def send(self, p, bufs, byte_idx=0):
        return self._send(p, bufs, byte_idx, self.pkg.ONE_CALL)

    def recv(self, p, cap):
        return self._recv(p, cap, self.pkg.ONE_CALL)

    def send_all(self, p, bufs, byte_idx=0):
        total = 0
        while True:
            n = self._send(p, bufs, byte_idx, self.pkg.UNTIL_BLOCKED)
            total += n
            window = sum(int(b.size) for b in bufs[:SLICE_AREA - 1]) - byte_idx
            if len(bufs) < SLICE_AREA or n < window:
                return total, -1
            bufs, byte_idx = bufs[SLICE_AREA - 1:], 0

    def recv_drain(self, p, cap):
        return self._recv(p, cap, self.pkg.UNTIL_BLOCKED), -1
