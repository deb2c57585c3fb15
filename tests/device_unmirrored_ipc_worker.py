"""One end of a CUDA-IPC / NVLink connection for tests/test_device_unmirrored_gpu.py.  The client claims its pair with
B200_CLAIM_UNMIRRORED, with or without the service running in its process: a device warp streams every message with
b200_warp_send (tests/native/device_poll.cu), b200_warp_poll waits for the frame the server sent, b200_warp_recv takes
it and b200_warp_disconnect closes the end.  Between the steps the client asks the host readiness and status queries
and runs b200_poller_scan on its end (without the service each query scans it); the end's PairMirror bytes must stay
those the claim left, and the queries must keep the answers they gave at the claim, until the release.  The server
sends that frame, receives with host calls, waits for HALF_CLOSED and stays until the client has released its end
(the client's status query probes whether this process still exists).  The two processes may share one GPU.

    python device_unmirrored_ipc_worker.py <role: client|server> <device> <dir> <ring_kb> <msg_bytes> <n_msgs> <service>
"""
import ctypes as C
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import __graft_entry__ as ge
from ipc_wire_worker import pattern, put_file, wait_file
from unmirrored_lib import mirror_bytes

HELLO = 777


def main():
    role, dev, d = sys.argv[1], int(sys.argv[2]), sys.argv[3]
    ring_kb, msg, n_msgs, service = int(sys.argv[4]), int(sys.argv[5]), int(sys.argv[6]), sys.argv[7] == "1"
    os.environ["B200_IPC_WIRE"] = "1"
    pkg = ge.load_package()
    pkg.init(dev)
    L = pkg.lib()
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", ring_kb)
    me, other = ("c", "s") if role == "client" else ("s", "c")
    p = pkg.Pair(me + "0")
    put_file(os.path.join(d, me + "0.addr"), p.address())
    assert p.connect(wait_file(os.path.join(d, other + "0.addr"))), p.error()
    hello = pattern(1, 0, HELLO)
    res = {"role": role}
    if role == "client":
        import device_poll_lib as dpl
        R = dpl.Runner(pkg)  # (the driver's kernels are loaded before the resident kernels start)
        if service:
            assert L.b200_service_start(4) == 0, pkg.last_error()
        arr = (C.c_void_p * 1)(p.h)
        scan_ev = np.zeros(1, np.uint32)

        def queries():
            L.b200_poller_scan(arr, 1, scan_ev.ctypes.data_as(C.POINTER(C.c_uint32)))
            return [p.status(), p.has_message(), p.readable(), p.writable(), p.has_pending_writes()]

        h = p.device_claim(mirrored=False)
        snap, at_claim = mirror_bytes(h), queries()
        frozen = [mirror_bytes(h) == snap]
        buf = L.b200_mem_alloc_device(msg)
        slp, sl = R.mem.array("slices", np.uint64, 2)
        sl[0], sl[1] = buf, msg
        ok = True
        for m in range(n_msgs):
            src = pattern(0, m, msg)
            assert L.b200_memcpy(buf, src.ctypes.data, msg, 0, None) == 0 and L.b200_stream_sync(None) == 0
            r = R.run([h], [[dict(kind=dpl.STREAM_SEND, pair=0, slices=slp, n=1)]], budget_s=120.0)[0][0]
            ok = ok and r["status"] == dpl.OK and r["ret"] == msg
            frozen.append(queries() == at_claim and mirror_bytes(h) == snap)
        res["ok"] = ok
        wait_file(os.path.join(d, "hello.sent"))
        evp, ev = R.mem.array("ev", np.uint32, 1)
        r = R.run([h], [[dict(kind=dpl.WAIT_EVENTS, pair=0, n=dpl.EV_READABLE, dst=evp)]], budget_s=60.0)[0][0]
        res["hello_seen"] = r["status"] == dpl.OK and bool(r["ret"] & dpl.EV_READABLE)
        frozen.append(queries() == at_claim and mirror_bytes(h) == snap)
        dstp, dst = R.mem.array("dst", np.uint8, 4096)
        r = R.run([h], [[dict(kind=dpl.STREAM_RECV, pair=0, dst=dstp, n=HELLO)]], budget_s=60.0)[0][0]
        res["hello_ok"] = r["status"] == dpl.OK and bool(np.array_equal(dst[:HELLO], hello))
        frozen.append(queries() == at_claim and mirror_bytes(h) == snap)
        res["closed"] = R.one(h, kind=dpl.DISCONNECT)
        frozen.append(queries() == at_claim and mirror_bytes(h) == snap)
        res["frozen"] = frozen
        res["at_claim"] = at_claim
        p.device_release()
        res["republished"] = mirror_bytes(h) != snap
        res["released"] = not p.device_owned() and p.status() == dpl.DISCONNECTED
        put_file(os.path.join(d, "client.released"), b"1")
        if service:
            L.b200_service_stop()
        L.b200_mem_free_device(buf)
        R.close()
    else:
        assert p.send([hello]) == HELLO
        put_file(os.path.join(d, "hello.sent"), b"1")
        total = msg * n_msgs
        host = np.zeros(total, np.uint8)
        got, t0 = 0, time.time()
        while got < total and time.time() - t0 < 120:
            n = L.b200_pair_recv(p.h, host.ctypes.data + got, total - got)
            got += n
            if n == 0:
                time.sleep(0.0005)
        res["drained"] = got
        res["ok"] = got == total and all(np.array_equal(host[m * msg:(m + 1) * msg], pattern(0, m, msg))
                                         for m in range(n_msgs))
        t0 = time.time()
        while p.status() != 3 and time.time() - t0 < 60:  # HALF_CLOSED once the client closed
            time.sleep(0.01)
        res["half_closed"] = p.status() == 3
        wait_file(os.path.join(d, "client.released"))  # (this process stays until then: the client probes it)
        p.disconnect()
    put_file(os.path.join(d, role + ".json"), json.dumps(res).encode())


if __name__ == "__main__":
    main()
