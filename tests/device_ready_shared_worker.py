"""The cases of tests/test_device_ready_shared_gpu.py, each in a process of its own.  TEST INFRASTRUCTURE.

    python device_ready_shared_worker.py <case>...

    traces-<mode>  random traces with 1 to 32 consumer warps and two consumer kernels (mode: reference, coalesced,
                   stamped)
    echo-<W>       an echo server of W warps on one set of 1024 claimed ends, 256 active device clients
    added          members added while an 8-warp consumer runs
Each case prints "case <x> ok" or "case <x> FAILED: <why>"; the exit status is 1 when one failed."""
import os
import sys
import traceback

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import __graft_entry__ as ge  # noqa: E402
import test_device_ready_shared_gpu as t  # noqa: E402


def main(cases):
    pkg = ge.load_package()
    pkg.init(0)
    failed = 0
    for case in cases:
        try:
            if case.startswith("traces-"):
                t.random_traces(pkg, case[len("traces-"):])
            elif case.startswith("echo-"):
                t.echo_server(pkg, int(case[len("echo-"):]))
            elif case == "added":
                t.members_added(pkg)
            else:
                raise ValueError("unknown case " + case)
            print("case %s ok" % case, flush=True)
        except Exception:
            failed = 1
            print("case %s FAILED: %s" % (case, traceback.format_exc()), flush=True)
    return failed


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
