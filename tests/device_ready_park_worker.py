"""The cases of tests/test_device_ready_park_gpu.py, each in a process of its own.  TEST INFRASTRUCTURE.

    python device_ready_park_worker.py <case>...

    host-park, one-ring, nonempty, add-disconnect-release, never-parked
    demand-<mode>-<svc|nosvc>-<warps>   launch on demand (mode: reference, coalesced, stamped)
Each case prints "case <x> ok" or "case <x> FAILED: <why>"; the exit status is 1 when one failed."""
import os
import sys
import traceback

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import __graft_entry__ as ge  # noqa: E402
import test_device_ready_park_gpu as t  # noqa: E402


def main(cases):
    pkg = ge.load_package()
    pkg.init(0)
    failed = 0
    for case in cases:
        try:
            t.run_case(pkg, case)
            print("case %s ok" % case, flush=True)
        except Exception:
            failed = 1
            print("case %s FAILED: %s" % (case, traceback.format_exc()), flush=True)
    return failed


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
