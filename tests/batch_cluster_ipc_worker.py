"""One end of a CUDA-IPC / NVLink connection whose sending end runs prepared-batch Sends with B200_BATCH_CLUSTER(K)
(tests/test_batch_cluster_gpu.py): the movers of K CTAs per op write the frames straight into the ring in the other
process's device memory, and the credit comes back over the wire.  The server receives with field-0 batches.  The two
processes may share one GPU.

    python batch_cluster_ipc_worker.py <K> <role: client|server> <device> <dir> <ring_kb> <msg_bytes> <n_msgs>
"""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import __graft_entry__ as ge  # noqa: E402
from ipc_wire_worker import pattern, put_file, wait_file  # noqa: E402


def main():
    k, role, dev, d = int(sys.argv[1]), sys.argv[2], int(sys.argv[3]), sys.argv[4]
    ring_kb, msg, n_msgs = int(sys.argv[5]), int(sys.argv[6]), int(sys.argv[7])
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
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(int)
        fl = pkg.UNTIL_BLOCKED | pkg.cluster_flag(k)
        ok, calls = True, []
        for m in range(n_msgs):
            src = pattern(0, m, total)
            assert L.b200_memcpy(buf, src.ctypes.data, total, 0, None) == 0 and L.b200_stream_sync(None) == 0
            idx = bidx = sent_total = n_calls = 0
            t0 = time.time()
            while idx < len(lens):
                sl = pkg.make_slices([(buf + int(offs[j]), lens[j]) for j in range(idx, len(lens))])
                bt = pkg.Batch("send", [(p, sl, len(lens) - idx, bidx)], fl)
                bt.launch()
                sent, c = bt.results()[0], bt.calls()[0]
                bt.destroy()
                sent_total += sent
                n_calls += c
                while sent > 0:
                    left = lens[idx] - bidx
                    if sent >= left:
                        sent, idx, bidx = sent - left, idx + 1, 0
                    else:
                        bidx, sent = bidx + sent, 0
                if time.time() - t0 > 120:
                    raise TimeoutError("message %d: sent %d of %d" % (m, sent_total, total))
            ok = ok and sent_total == total
            calls.append(n_calls)
        res["ok"] = ok
        res["calls"] = calls
        res["pending"] = p.has_pending_writes()
        res["state"] = p.state()
        wait_file(os.path.join(d, "server.done"))
        p.disconnect()
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
    L.b200_mem_free_device(buf)
    put_file(os.path.join(d, role + ".json"), json.dumps(res).encode())


if __name__ == "__main__":
    main()
