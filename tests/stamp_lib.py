"""ctypes loader for the stamped ring frame model (tests/native/stamp_oracle.c).  TEST INFRASTRUCTURE.

`StampedOracle` is orlib.Oracle with Send / Recv / readiness replaced by the stamped ones, so that
tests/trace.run_trace replays a trace under B200_RING_STAMPED=1 semantics on the CPU (coalesced=True: with
B200_SEND_COALESCE=1 as well)."""
import ctypes as C
import os
import subprocess

import numpy as np

import orlib

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
LIB = os.path.join(NATIVE, "libstamp_oracle.so")


def load():
    if not os.path.exists(os.path.join(orlib.ORACLE_DIR, "liboracle.so")):
        orlib.build_oracle()
    subprocess.check_call(["make", "-s", "-C", NATIVE, "-f", "stamp.mk"])
    L = C.CDLL(LIB)
    u64, P, S = C.c_uint64, C.POINTER(orlib.OrbPair), C.POINTER(orlib.Slice)
    for name, res, args in [
        ("stamp_of", C.c_uint32, [u64]), ("stamp_header", u64, [u64, u64]),
        ("stamp_seq_set", None, [P, u64, u64]), ("stamp_seq_tx", u64, [P]), ("stamp_seq_rx", u64, [P]),
        ("stamp_forget", None, [P]), ("stamp_pads", C.c_void_p, [P]),
        ("stamp_readable", u64, [P]), ("stamp_has_message", C.c_int, [P]), ("stamp_pair_readable", u64, [P]),
        ("stamp_recv", u64, [P, C.c_void_p, u64]), ("stamp_recv_drain", u64, [P, C.c_void_p, u64, C.POINTER(u64)]),
        ("stamp_send", u64, [P, S, C.c_size_t, C.c_size_t]),
        ("stamp_send_coalesced", u64, [P, S, C.c_size_t, C.c_size_t]),
        ("stamp_send_all", u64, [P, S, C.c_size_t, C.c_size_t, C.c_int, C.POINTER(u64)]),
        ("stamp_ops_config", None, [u64]), ("stamp_pair_ops", C.c_void_p, []), ("stamp_pair_ops_batch", C.c_void_p, []),
    ]:
        f = getattr(L, name)
        f.restype, f.argtypes = res, args
    return L


class StampedOracle(orlib.Oracle):
    kind = "port-stamped"

    def __init__(self, coalesced=False):
        super().__init__()
        self.S = load()
        self.coalesced = coalesced

    def pair_pair(self, cap, max_sge=30):
        a, b = super().pair_pair(cap, max_sge)
        for p in (a, b):
            self.S.stamp_seq_set(p, 0, 0)
        return a, b

    def destroy(self, p):
        self.S.stamp_forget(p)
        super().destroy(p)

    def send(self, p, bufs, byte_idx=0):
        f = self.S.stamp_send_coalesced if self.coalesced else self.S.stamp_send
        return f(p, orlib.make_slices(bufs), len(bufs), byte_idx)

    def send_all(self, p, bufs, byte_idx=0):
        calls = C.c_uint64(0)
        n = self.S.stamp_send_all(p, orlib.make_slices(bufs), len(bufs), byte_idx, int(self.coalesced), C.byref(calls))
        return n, calls.value

    def recv(self, p, cap):
        out = np.zeros(max(cap, 1), dtype=np.uint8)
        n = self.S.stamp_recv(p, out.ctypes.data, cap)
        return out[:n].copy()

    def recv_drain(self, p, cap):
        out = np.zeros(max(cap, 1), dtype=np.uint8)
        calls = C.c_uint64(0)
        n = self.S.stamp_recv_drain(p, out.ctypes.data, cap, C.byref(calls))
        return out[:n].copy(), calls.value

    def pads(self, p):
        """bool mask of the pad bytes in p's ring image"""
        cap = p.contents.ring.capacity
        return np.ctypeslib.as_array((C.c_uint8 * cap).from_address(self.S.stamp_pads(p))).astype(bool)

    def has_message(self, p):
        return int(self.S.stamp_has_message(p))

    def readable(self, p):
        return self.S.stamp_pair_readable(p)

