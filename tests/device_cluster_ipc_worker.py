"""One end of a CUDA-IPC / NVLink connection whose sending end is driven from a user kernel's thread-block cluster
(tests/test_device_cluster_gpu.py).  The roles are those of device_block_ipc_worker.py, with the client's
STREAM_SEND ops run by clusters of K CTAs through b200_cluster_send (tests/native/device_cluster.cu): the frames go
from the movers of K CTAs straight into the ring in the other process's device memory and the credit comes back over
the wire.

    python device_cluster_ipc_worker.py <K> <role: client|server> <device> <dir> <ring_kb> <msg_bytes> <n_msgs>
"""
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import device_block_ipc_worker  # noqa: E402
import device_cluster_lib  # noqa: E402


def main():
    k = int(sys.argv[1])
    # the block worker's client takes Runner, STREAM_SEND and OK from device_block_lib: hand it the cluster driver's
    adapter = types.ModuleType("device_block_lib")
    adapter.Runner = lambda pkg: device_cluster_lib.Runner(pkg, k)
    adapter.STREAM_SEND, adapter.OK = device_cluster_lib.STREAM_SEND, device_cluster_lib.OK
    sys.modules["device_block_lib"] = adapter
    sys.argv = sys.argv[:1] + sys.argv[2:]
    device_block_ipc_worker.main()


if __name__ == "__main__":
    main()
