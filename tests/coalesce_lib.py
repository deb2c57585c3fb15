"""ctypes loader for the coalesced-Send model (tests/native/coalesce_oracle.c).  TEST INFRASTRUCTURE.

`CoalescedOracle` is orlib.Oracle with Send / the rdma_flush loop replaced by the coalesced ones, so that
tests/trace.run_trace replays a trace under B200_SEND_COALESCE=1 semantics on the CPU."""
import ctypes as C
import os
import subprocess

import orlib

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
LIB = os.path.join(NATIVE, "libcoalesce_oracle.so")


def load():
    if not os.path.exists(os.path.join(orlib.ORACLE_DIR, "liboracle.so")):
        orlib.build_oracle()
    subprocess.check_call(["make", "-s", "-C", NATIVE, "-f", "coalesce.mk"])
    L = C.CDLL(LIB)
    u64, P = C.c_uint64, C.POINTER(orlib.OrbPair)
    L.orb_pair_send_coalesced.restype = u64
    L.orb_pair_send_coalesced.argtypes = [P, C.POINTER(orlib.Slice), C.c_size_t, C.c_size_t]
    L.orb_pair_send_coalesced_all.restype = u64
    L.orb_pair_send_coalesced_all.argtypes = [P, C.POINTER(orlib.Slice), C.c_size_t, C.c_size_t, C.POINTER(u64)]
    L.coalesce_ops_config.argtypes = [u64]
    L.coalesce_pair_ops.restype = C.c_void_p
    L.coalesce_pair_ops_batch.restype = C.c_void_p
    return L


class CoalescedOracle(orlib.Oracle):
    kind = "port-coalesced"

    def __init__(self):
        super().__init__()
        self.C = load()

    def send(self, p, bufs, byte_idx=0):
        return self.C.orb_pair_send_coalesced(p, orlib.make_slices(bufs), len(bufs), byte_idx)

    def send_all(self, p, bufs, byte_idx=0):
        calls = C.c_uint64(0)
        n = self.C.orb_pair_send_coalesced_all(p, orlib.make_slices(bufs), len(bufs), byte_idx, C.byref(calls))
        return n, calls.value


def chttp2_lens(data):
    """chttp2's slicing of a gRPC message of `data` bytes (+5-byte prefix): 9-byte DATA headers, <= 16 KiB payloads."""
    lens, data = [], data + 5
    while data > 0:
        n = min(16384, data)
        lens += [9, n]
        data -= n
    return lens
