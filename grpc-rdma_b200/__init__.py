"""grpc-rdma_b200 -- GPU-native (H100, sm_90a) RDMA_BPEV endpoint hot path (host-side Python binding).

The product is the C-ABI shared library ``lib/libb200rdma.so`` declared in
``include/b200_pair.h`` (CUDA kernels + host runtime under ``csrc/``).  This
module is only a ctypes binding used by tests and ``bench.py``; it mirrors the
reference's PairPollable surface (src/core/lib/ibverbs/pair.h:82-271) name by
name.  There is no CPU fallback: importing works without a GPU (so the symbol
table can be checked), but every data-path call fails loudly if the library or
a CUDA device is missing.

The directory name contains a hyphen, so load it with
``__graft_entry__.load_package()`` (registers it as ``grpc_rdma_b200``).
"""
import ctypes as C
import numbers
import os
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG_DIR)
LIB_PATH = os.environ.get("B200RDMA_LIB") or os.path.join(PKG_DIR, "lib", "libb200rdma.so")  # env: experiment builds
HEADER = os.path.join(ROOT, "include", "b200_pair.h")
ENDPOINT_LIB_PATH = os.path.join(PKG_DIR, "lib", "libb200_endpoint.so")
ENDPOINT_HEADER = os.path.join(ROOT, "include", "b200_endpoint.h")

ADDRESS_BYTES = 48
DEV_PAIR_BYTES = 64  # sizeof(b200_dev_pair)
DEV_READY_SET_BYTES = 64  # sizeof(b200_dev_ready_set)
CLAIM_UNMIRRORED = 0x1  # B200_CLAIM_UNMIRRORED (b200_pair_device_claim_ex)
ONE_CALL, UNTIL_BLOCKED, ASYNC, ZEROCOPY = 0, 1, 2, 4
EV_READABLE, EV_WRITABLE = 0x1, 0x4
STATUS = ["UNINITIALIZED", "INITIALIZED", "CONNECTED", "HALF_CLOSED", "DISCONNECTED", "ERROR"]


def cluster_flag(k):
    """B200_BATCH_CLUSTER(k): batch flag bits that run each op on a thread-block cluster of k CTAs (1 <= k <= 16;
    k = 1 is the default, one CTA per op)."""
    if isinstance(k, bool) or not isinstance(k, numbers.Integral) or not 1 <= k <= 16:
        raise ValueError("cluster width must be an integer in 1..16, got %r" % (k,))
    return (int(k) - 1) << 4


class Slice(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("len", C.c_uint64)]


class SendOp(C.Structure):
    _fields_ = [("pair", C.c_void_p), ("slices", C.POINTER(Slice)), ("nslices", C.c_size_t),
                ("byte_idx", C.c_size_t)]


class RecvOp(C.Structure):
    _fields_ = [("pair", C.c_void_p), ("dst", C.c_void_p), ("cap", C.c_uint64)]


class PairState(C.Structure):
    _fields_ = [("head", C.c_uint64), ("moving_head", C.c_uint64), ("remain", C.c_uint64),
                ("remote_tail", C.c_uint64), ("internal_read_size", C.c_uint64),
                ("credit_remote_head", C.c_uint64), ("partial_write", C.c_uint32), ("peer_exit", C.c_uint32),
                ("ring_capacity", C.c_uint64)]


def build(verbose=False):
    """Compile lib/libb200rdma.so for sm_90a (nvcc cross-compiles without a GPU)."""
    out = subprocess.run(["make", "-C", PKG_DIR, "all"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("building libb200rdma.so failed:\n" + out.stdout + out.stderr)
    if verbose:
        print(out.stdout + out.stderr)
    return LIB_PATH


_SIGS = {
    # name: (restype, argtypes)
    "b200_init": (C.c_int, [C.c_int]),
    "b200_shutdown": (None, []),
    "b200_device": (C.c_int, []),
    "b200_last_error": (C.c_char_p, []),
    "b200_config_set": (C.c_int, [C.c_char_p, C.c_char_p]),
    "b200_config_get": (C.c_int64, [C.c_char_p]),
    "b200_mem_alloc_device": (C.c_void_p, [C.c_size_t]),
    "b200_mem_free_device": (None, [C.c_void_p]),
    "b200_mem_alloc_host": (C.c_void_p, [C.c_size_t]),
    "b200_mem_free_host": (None, [C.c_void_p]),
    "b200_mem_register_host": (C.c_int, [C.c_void_p, C.c_size_t]),
    "b200_mem_unregister_host": (C.c_int, [C.c_void_p]),
    "b200_memcpy": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "b200_stream_sync": (C.c_int, [C.c_void_p]),
    "b200_pool_take": (C.c_void_p, [C.c_char_p]),
    "b200_pool_putback": (None, [C.c_void_p]),
    "b200_pool_get": (C.c_void_p, [C.c_char_p]),
    "b200_pair_init": (None, [C.c_void_p]),
    "b200_pair_self_address": (C.c_size_t, [C.c_void_p, C.c_void_p]),
    "b200_pair_connect": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "b200_pair_disconnect": (None, [C.c_void_p]),
    "b200_pair_send": (C.c_uint64, [C.c_void_p, C.POINTER(Slice), C.c_size_t, C.c_size_t]),
    "b200_pair_recv": (C.c_uint64, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "b200_pair_has_message": (C.c_int, [C.c_void_p]),
    "b200_pair_has_pending_writes": (C.c_int, [C.c_void_p]),
    "b200_pair_readable": (C.c_uint64, [C.c_void_p]),
    "b200_pair_writable": (C.c_uint64, [C.c_void_p]),
    "b200_pair_status": (C.c_int, [C.c_void_p]),
    "b200_pair_error": (C.c_char_p, [C.c_void_p]),
    "b200_pair_stamped": (C.c_int, [C.c_void_p]),
    "b200_pair_wakeup_read_fd": (C.c_int, [C.c_void_p]),
    "b200_pair_consume_wakeup": (None, [C.c_void_p]),
    "b200_pair_get_state": (C.c_int, [C.c_void_p, C.POINTER(PairState)]),
    "b200_pair_copy_ring": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "b200_poller_add": (None, [C.c_void_p]),
    "b200_poller_remove": (None, [C.c_void_p]),
    "b200_poller_shutdown": (None, []),
    "b200_poller_scan": (C.c_int, [C.POINTER(C.c_void_p), C.c_size_t, C.POINTER(C.c_uint32)]),
    "b200_service_start": (C.c_int, [C.c_int]),
    "b200_service_stop": (None, []),
    "b200_service_running": (C.c_int, []),
    "b200_service_stats": (None, [C.POINTER(C.c_uint64)]),
    "b200_service_eager_hits": (C.c_uint64, []),
    "b200_pairs_send": (C.c_int, [C.POINTER(SendOp), C.c_size_t, C.c_int, C.POINTER(C.c_uint64), C.c_void_p]),
    "b200_pairs_recv": (C.c_int, [C.POINTER(RecvOp), C.c_size_t, C.c_int, C.POINTER(C.c_uint64), C.c_void_p]),
    "b200_pairs_submit": (C.c_int, [C.POINTER(SendOp), C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(RecvOp), C.c_size_t,
                                    C.POINTER(C.c_uint64), C.c_int]),
    "b200_pair_post_send": (C.c_void_p, [C.c_void_p, C.POINTER(Slice), C.c_size_t, C.c_size_t, C.c_int, C.POINTER(C.c_int)]),
    "b200_pair_post_recv": (C.c_void_p, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(C.c_int)]),
    "b200_async_poll": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "b200_batch_prepare_send": (C.c_void_p, [C.POINTER(SendOp), C.c_size_t, C.c_int]),
    "b200_batch_prepare_recv": (C.c_void_p, [C.POINTER(RecvOp), C.c_size_t, C.c_int]),
    "b200_batch_launch": (C.c_int, [C.c_void_p, C.c_void_p]),
    "b200_batch_results": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p]),
    "b200_lanes_fork": (C.c_int, [C.c_void_p]),
    "b200_lanes_join": (C.c_int, [C.c_void_p]),
    "b200_batch_calls": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "b200_batch_destroy": (None, [C.c_void_p]),
    "b200_probe_copy": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_uint32,
                                  C.c_uint32, C.c_uint32, C.c_void_p]),
    "b200_launch_count": (C.c_uint64, []),
    "b200_pair_device_claim": (C.c_int, [C.c_void_p, C.c_void_p]),
    "b200_pair_device_claim_ex": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "b200_pair_device_release": (C.c_int, [C.c_void_p]),
    "b200_pair_device_owned": (C.c_int, [C.c_void_p]),
    "b200_ready_set_create": (C.c_void_p, [C.c_uint32]),
    "b200_ready_set_device": (C.c_int, [C.c_void_p, C.c_void_p]),
    "b200_ready_set_destroy": (C.c_int, [C.c_void_p]),
    "b200_ready_set_add": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32]),
    "b200_ready_set_park": (C.c_int, [C.c_void_p]),
    "b200_ready_set_wakeup_fd": (C.c_int, [C.c_void_p]),
    "b200_ready_set_consume_wakeup": (None, [C.c_void_p]),
    "b200_ready_set_rings": (C.c_uint64, [C.c_void_p]),
}

_lib = None


def exported_symbols():
    """Names the header declares (every `b200_*(` prototype)."""
    import re
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", txt)))


def lib():
    """Load the C-ABI library (no CPU fallback: raises if it is not built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libb200rdma.so is not built (run __graft_entry__.build()); there is no CPU fallback for this path")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            f = getattr(L, name)
            f.restype = res
            f.argtypes = args
        _lib = L
    return _lib


def last_error():
    return lib().b200_last_error().decode()


def init(device=-1):
    if lib().b200_init(device) != 0:
        raise RuntimeError("b200_init failed: " + last_error())


def config_set(key, value):
    if lib().b200_config_set(key.encode(), str(value).encode()) != 0:
        raise ValueError("b200_config_set(%s=%s) rejected: %s" % (key, value, last_error()))


def make_slices(ptr_len_list):
    arr = (Slice * max(1, len(ptr_len_list)))()
    for i, (p, n) in enumerate(ptr_len_list):
        arr[i].ptr = p
        arr[i].len = n
    return arr


class Pair:
    """Mirror of grpc_core::ibverbs::PairPollable over the C ABI."""

    def __init__(self, ident=""):
        self.L = lib()
        self.h = self.L.b200_pool_take(ident.encode())
        if not self.h:
            raise RuntimeError("b200_pool_take failed: " + last_error())
        self.L.b200_pair_init(self.h)
        if self.L.b200_pair_status(self.h) != 1:
            raise RuntimeError("b200_pair_init failed: " + self.L.b200_pair_error(self.h).decode())

    def address(self):
        buf = C.create_string_buffer(ADDRESS_BYTES)
        n = self.L.b200_pair_self_address(self.h, buf)
        return buf.raw[:n]

    def connect(self, peer_bytes):
        return self.L.b200_pair_connect(self.h, peer_bytes, len(peer_bytes)) == 1

    def send(self, np_bufs, byte_idx=0):
        sl = make_slices([(b.ctypes.data if b.size else 0, b.size) for b in np_bufs])
        return self.L.b200_pair_send(self.h, sl, len(np_bufs), byte_idx)

    def send_raw(self, ptr_len_list, byte_idx=0):
        return self.L.b200_pair_send(self.h, make_slices(ptr_len_list), len(ptr_len_list), byte_idx)

    def recv(self, cap):
        import numpy as np
        out = np.zeros(max(cap, 1), dtype=np.uint8)
        n = self.L.b200_pair_recv(self.h, out.ctypes.data, cap)
        return out[:n].copy()

    def recv_into(self, ptr, cap):
        return self.L.b200_pair_recv(self.h, ptr, cap)

    def has_message(self):
        return self.L.b200_pair_has_message(self.h)

    def has_pending_writes(self):
        return self.L.b200_pair_has_pending_writes(self.h)

    def readable(self):
        return self.L.b200_pair_readable(self.h)

    def writable(self):
        return self.L.b200_pair_writable(self.h)

    def status(self):
        return self.L.b200_pair_status(self.h)

    def error(self):
        return self.L.b200_pair_error(self.h).decode()

    def stamped(self):
        """True when the connected pair runs stamped ring frames (both ends offered B200_RING_STAMPED)."""
        return self.L.b200_pair_stamped(self.h) == 1

    def wakeup_fd(self):
        return self.L.b200_pair_wakeup_read_fd(self.h)

    def state(self):
        st = PairState()
        if self.L.b200_pair_get_state(self.h, C.byref(st)) != 0:
            raise RuntimeError(last_error())
        return dict(head=st.head, moving_head=st.moving_head, remain=st.remain, remote_tail=st.remote_tail,
                    internal_read_size=st.internal_read_size, partial_write=int(st.partial_write),
                    credit_remote_head=st.credit_remote_head, peer_exit=int(st.peer_exit))

    def ring_image(self):
        import numpy as np
        st = PairState()
        self.L.b200_pair_get_state(self.h, C.byref(st))
        out = np.zeros(st.ring_capacity, dtype=np.uint8)
        if self.L.b200_pair_copy_ring(self.h, out.ctypes.data, out.size) != 0:
            raise RuntimeError(last_error())
        return out

    def device_claim(self, mirrored=True):
        """Hand this end to the caller's kernels (include/b200_device.cuh): returns the 64-byte b200_dev_pair
        handle.  Host calls on this end are refused until device_release().  mirrored=False claims it with
        B200_CLAIM_UNMIRRORED: nothing writes its host-visible mirror until the release, so its host readiness and
        status queries stay as the claim left them."""
        buf = C.create_string_buffer(DEV_PAIR_BYTES)
        if mirrored:
            rc = self.L.b200_pair_device_claim(self.h, buf)
        else:
            rc = self.L.b200_pair_device_claim_ex(self.h, CLAIM_UNMIRRORED, buf)
        if rc != 0:
            raise RuntimeError("b200_pair_device_claim failed: " + last_error())
        return buf.raw

    def device_release(self):
        """Give the end back to the host; the kernels that used the handle must have finished."""
        if self.L.b200_pair_device_release(self.h) != 0:
            raise RuntimeError("b200_pair_device_release failed: " + last_error())

    def device_owned(self):
        return self.L.b200_pair_device_owned(self.h) == 1

    def disconnect(self):
        self.L.b200_pair_disconnect(self.h)

    def putback(self):
        self.L.b200_pool_putback(self.h)


class ReadySet:
    """A device ready set (b200_ready_set_*): the queue consumer warps take ready members' keys from
    (include/b200_device.cuh: b200_warp_ready_take / b200_warp_ready_rearm).  Any number of warps, in one kernel or
    in several, may take from one set; each entry goes to one warp, which holds that member until its rearm returns 0.
    Members are claimed Pairs on the loopback wire; membership ends with the claim.  A parked set (park(), or
    b200_warp_ready_park in a kernel) rings its doorbell at the next entry; the Poller then kicks wakeup_fd()."""

    def __init__(self, capacity):
        self.L = lib()
        self.h = self.L.b200_ready_set_create(capacity)
        if not self.h:
            raise RuntimeError("b200_ready_set_create failed: " + last_error())

    def device(self):
        """the 64-byte b200_dev_ready_set handle for kernels"""
        buf = C.create_string_buffer(DEV_READY_SET_BYTES)
        if self.L.b200_ready_set_device(self.h, buf) != 0:
            raise RuntimeError(last_error())
        return buf.raw

    def add(self, pair, key):
        """make the claimed `pair` a member with `key`; raises with b200_last_error's reason when refused"""
        if self.L.b200_ready_set_add(self.h, pair.h, key) != 0:
            raise RuntimeError("b200_ready_set_add failed: " + last_error())

    def park(self):
        """park the set from the host (no consumer may be taking): 0 parked, the next entry queued rings the
        doorbell; 1 entries are queued, launch a server; raises on failure"""
        rc = self.L.b200_ready_set_park(self.h)
        if rc < 0:
            raise RuntimeError("b200_ready_set_park failed: " + last_error())
        return rc

    def wakeup_fd(self):
        """the set's eventfd, kicked by the Poller when the doorbell rings (the first call registers the set)"""
        fd = self.L.b200_ready_set_wakeup_fd(self.h)
        if fd < 0:
            raise RuntimeError("b200_ready_set_wakeup_fd failed: " + last_error())
        return fd

    def consume_wakeup(self):
        self.L.b200_ready_set_consume_wakeup(self.h)

    def rings(self):
        """doorbell rings so far: one per park that a later entry answered"""
        return self.L.b200_ready_set_rings(self.h)

    def destroy(self):
        """no kernel may use the set; raises while it has members"""
        if self.L.b200_ready_set_destroy(self.h) != 0:
            raise RuntimeError("b200_ready_set_destroy failed: " + last_error())
        self.h = None


def connected_pair(ident_a="a", ident_b="b"):
    a, b = Pair(ident_a), Pair(ident_b)
    if not a.connect(b.address()) or not b.connect(a.address()):
        raise RuntimeError("connect failed: %s / %s" % (a.error(), b.error()))
    return a, b


class Batch:
    """Prepared batch (descriptors resident in HBM), see b200_batch_* in the header."""

    def __init__(self, kind, ops, flags):
        L = self.L = lib()
        self.n = len(ops)
        self._keep = ops
        if kind == "send":
            arr = (SendOp * max(1, self.n))()
            for i, (pair, sl, nsl, bidx) in enumerate(ops):
                arr[i].pair, arr[i].slices, arr[i].nslices, arr[i].byte_idx = pair.h, sl, nsl, bidx
            self.h = L.b200_batch_prepare_send(arr, self.n, flags)
        else:
            arr = (RecvOp * max(1, self.n))()
            for i, (pair, dst, cap) in enumerate(ops):
                arr[i].pair, arr[i].dst, arr[i].cap = pair.h, dst, cap
            self.h = L.b200_batch_prepare_recv(arr, self.n, flags)
        if not self.h:
            raise RuntimeError("b200_batch_prepare failed: " + last_error())

    def launch(self, stream=None):
        if self.L.b200_batch_launch(self.h, stream) != 0:
            raise RuntimeError("b200_batch_launch failed: " + last_error())

    def results(self, stream=None):
        out = (C.c_uint64 * max(1, self.n))()
        if self.L.b200_batch_results(self.h, out, stream) != 0:
            raise RuntimeError("b200_batch_results failed: " + last_error())
        return list(out)[:self.n]

    def calls(self):
        out = (C.c_uint64 * max(1, self.n))()
        self.L.b200_batch_calls(self.h, out)
        return list(out)[:self.n]

    def destroy(self):
        if self.h:
            self.L.b200_batch_destroy(self.h)
            self.h = None


# --------------------------------------------------------------------------
# Workload shapes (SURVEY.md section 8d): how chttp2 hands a gRPC message to
# the endpoint -- alternating 9-byte HTTP/2 DATA frame headers and <= 16384-byte
# payload slices (src/core/ext/transport/chttp2/transport/frame_data.cc:64-...,
# writing.cc:191-193), the first payload slice prefixed by the 5-byte gRPC
# message header.
# --------------------------------------------------------------------------
HTTP2_MAX_FRAME = 16384


def chttp2_slice_lens(message_bytes, max_frame=HTTP2_MAX_FRAME):
    data = 5 + message_bytes
    lens = []
    while data > 0:
        n = min(max_frame, data)
        lens += [9, n]
        data -= n
    return lens


def frame_hbm_bytes(lens, stamped=False):
    """Algorithmic HBM bytes for one pass of the slice list (DESIGN.md):
    gather reads p and writes E(p); deframe reads E, writes p, clears E
    (stamped ring frames: reads E, writes p, no clear)."""
    tx = rx = 0
    for p in lens:
        e = 16 + ((p + 7) // 8) * 8
        tx += p + e
        rx += e + p + (0 if stamped else e)
    return tx, rx
