"""Trace adapters whose claimed ends are claimed with B200_CLAIM_UNMIRRORED (b200_pair_device_claim_ex), and the
PairMirror bytes of a claimed end.  TEST INFRASTRUCTURE."""
import ctypes as C
import struct

import device_block_lib as bl
import device_cluster_lib as cl
import device_lib
from device_lib import DeviceEngine

MIRROR_BYTES = 72  # sizeof(PairMirror), grpc-rdma_b200/csrc/b200_dev.cuh


def mirror_bytes(handle):
    """the end's PairMirror (pinned host memory): the handle's `mirrors` base, row `slot`"""
    base = struct.unpack_from("<Q", handle, 16)[0]
    slot = struct.unpack_from("<i", handle, 24)[0]
    return C.string_at(base + MIRROR_BYTES * slot, MIRROR_BYTES)


def writable_size(cap, head, tail):  # GetWritableSize, ring_buffer.cc:106-116
    f = cap - ((tail + cap - head) & (cap - 1))
    return f - 24 if f > 24 else 0


class Unmirrored:
    """Mixin for the device trace engines: the claimed ends named in `unmirrored` are claimed with
    B200_CLAIM_UNMIRRORED.  Their readiness answers come from the device (b200_warp_readable / has_message /
    has_pending_writes through the warp driver, GetWritableSize from get_state): the host queries of such an end are
    frozen.  Every query and every op checks that the mirror bytes of every unmirrored end are those the claim left;
    at destroy the end is released and its host queries must equal the device's answers from just before."""

    def __init__(self, *a, unmirrored=("tx", "rx"), **kw):
        super().__init__(*a, **kw)
        self.unmirrored = unmirrored
        self.frozen = {}

    def pair_pair(self, cap, max_sge=30):
        tx, rx = super().pair_pair(cap, max_sge)
        self.cap = cap
        for name, p in (("tx", tx), ("rx", rx)):
            if p.h in self.handles and name in self.unmirrored:
                p.device_release()
                h = p.device_claim(mirrored=False)
                self.handles[p.h] = h
                self.frozen[p.h] = (h, mirror_bytes(h))
        return tx, rx

    def check_frozen(self):
        for h, snap in self.frozen.values():
            assert mirror_bytes(h) == snap, "a library write reached an unmirrored end's PairMirror"

    def _device_answers(self, p):
        r = self.R.run([self.handles[p.h]], [[dict(kind=device_lib.READY, pair=0)]])[0][0]
        assert r["status"] == device_lib.OK, r
        st = p.state()
        return dict(readable=r["ret"], has_message=r["calls"] & 1, pending=r["calls"] >> 1,
                    writable=writable_size(self.cap, st["credit_remote_head"], st["remote_tail"]))

    def _answer(self, p, key, host):
        self.check_frozen()
        if p.h in self.frozen:
            return self._device_answers(p)[key]
        return host(p)

    def has_message(self, p):
        return self._answer(p, "has_message", super().has_message)

    def readable(self, p):
        return self._answer(p, "readable", super().readable)

    def has_pending_writes(self, p):
        return self._answer(p, "pending", super().has_pending_writes)

    def writable(self, p):
        return self._answer(p, "writable", super().writable)

    def state(self, p):
        self.check_frozen()
        return super().state(p)

    def destroy(self, p):
        if p.h in self.frozen:
            self.check_frozen()
            want = self._device_answers(p)
            self.frozen.pop(p.h)
            self.handles.pop(p.h)
            p.device_release()
            got = dict(readable=p.readable(), has_message=p.has_message(), pending=p.has_pending_writes(),
                       writable=p.writable())
            assert got == want, (got, want)
        super().destroy(p)


class UnmirroredDeviceEngine(Unmirrored, DeviceEngine):
    kind = "device-unmirrored"


class UnmirroredBlockEngine(Unmirrored, bl.BlockEngine):
    kind = "block-unmirrored"


class UnmirroredClusterEngine(Unmirrored, cl.ClusterEngine):
    kind = "cluster-unmirrored"


def engines(gpu, kind, mem="device", mis=0, **kw):
    """(mirrored, unmirrored) twin engines of one kind: "warp", "block", "cluster2", "cluster4" """
    um = kw.pop("unmirrored", ("tx", "rx"))
    if kind == "warp":
        return DeviceEngine(gpu, mem, mis, **kw), UnmirroredDeviceEngine(gpu, mem, mis, unmirrored=um, **kw)
    if kind == "block":
        return bl.BlockEngine(gpu, mem, mis, **kw), UnmirroredBlockEngine(gpu, mem, mis, unmirrored=um, **kw)
    k = int(kind[len("cluster"):])
    return cl.ClusterEngine(gpu, k, mem, mis, **kw), UnmirroredClusterEngine(gpu, k, mem, mis, unmirrored=um, **kw)
