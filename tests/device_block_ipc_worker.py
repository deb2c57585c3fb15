"""One end of a CUDA-IPC / NVLink connection whose sending end is driven from a user kernel's CTA
(tests/test_device_block_gpu.py): the client claims its pair and streams every message with b200_block_send
(tests/native/device_block.cu), so the frames go from the bulk-copy movers of a device CTA straight into the ring in the
other process's device memory and the credit comes back over the wire; the server receives with host batches.  The
two processes may share one GPU.

    python device_block_ipc_worker.py <role: client|server> <device> <dir> <ring_kb> <msg_bytes> <n_msgs>
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


def main():
    role, dev, d = sys.argv[1], int(sys.argv[2]), sys.argv[3]
    ring_kb, msg, n_msgs = int(sys.argv[4]), int(sys.argv[5]), int(sys.argv[6])
    os.environ["B200_IPC_WIRE"] = "1"
    pkg = ge.load_package()
    pkg.init(dev)
    L = pkg.lib()
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", ring_kb)
    me, other = ("c", "s") if role == "client" else ("s", "c")
    p = pkg.Pair(me + "0")
    put_file(os.path.join(d, me + "0.addr"), p.address())
    assert p.connect(wait_file(os.path.join(d, other + "0.addr"))), p.error()
    lens = pkg.chttp2_slice_lens(msg)
    total = sum(lens)
    buf = L.b200_mem_alloc_device(total)
    res = {"role": role}
    if role == "client":
        import device_block_lib as device_lib
        R = device_lib.Runner(pkg)
        h = p.device_claim()
        slp = L.b200_mem_alloc_host(16 * len(lens))
        arr = (pkg.Slice * len(lens)).from_address(slp)
        off = 0
        for k, n in enumerate(lens):
            arr[k].ptr, arr[k].len = buf + off, n
            off += n
        sent = []
        for m in range(n_msgs):
            src = pattern(0, m, total)
            assert L.b200_memcpy(buf, src.ctypes.data, total, 0, None) == 0 and L.b200_stream_sync(None) == 0
            r = R.run([h], [[dict(kind=device_lib.STREAM_SEND, pair=0, slices=slp, n=len(lens))]], budget_s=120.0)
            sent.append(r[0][0])
        res["ok"] = all(s["status"] == device_lib.OK and s["ret"] == total for s in sent)
        res["calls"] = [s["calls"] for s in sent]
        res["pending"] = p.has_pending_writes()
        res["state"] = p.state()
        wait_file(os.path.join(d, "server.done"))
        p.disconnect()  # releases the claim; the server sees peer_exit
        res["released"] = not p.device_owned()
    else:
        host = np.zeros(total, np.uint8)
        ok = True
        for m in range(n_msgs):
            got, t0 = 0, time.time()
            while got < total:
                bt = pkg.Batch("recv", [(p, buf + got, total - got)], pkg.UNTIL_BLOCKED)
                bt.launch(None)
                got += bt.results(None)[0]
                bt.destroy()
                if time.time() - t0 > 120:
                    raise TimeoutError("message %d: got %d of %d" % (m, got, total))
            assert L.b200_memcpy(host.ctypes.data, buf, total, 1, None) == 0 and L.b200_stream_sync(None) == 0
            ok = ok and bool(np.array_equal(host, pattern(0, m, total)))
        res["ok"] = ok
        res["state"] = p.state()
        res["ring_empty"] = bool(not p.ring_image().any())
        put_file(os.path.join(d, "server.done"), b"1")
        t0 = time.time()
        while p.status() != 3 and time.time() - t0 < 30:  # HALF_CLOSED once the client left
            time.sleep(0.01)
        res["half_closed"] = p.status() == 3
        p.disconnect()
    put_file(os.path.join(d, role + ".json"), json.dumps(res).encode())


if __name__ == "__main__":
    main()
