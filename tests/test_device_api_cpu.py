"""CPU: the device API (include/b200_device.cuh) and its test driver compile for sm_90a against the public header
alone, the driver's kernel does not spill, and the library exports the claim / release calls.  No GPU needed."""
import os
import re
import subprocess
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

# a user kernel: nothing but the public header and the ABI header it includes
USER_KERNEL = r'''
#include "b200_device.cuh"
__global__ void echo(const b200_dev_pair* tx, const b200_dev_pair* rx, const b200_slice* s, uint32_t n, uint8_t* dst,
                     uint64_t* out) {
  const uint64_t sent = b200_warp_send(tx, s, n, 0);
  const uint64_t got = b200_warp_recv(rx, dst, sent);
  if ((threadIdx.x & 31) == 0)
    out[0] = sent + got + b200_warp_readable(rx) + b200_warp_has_message(rx) + b200_warp_has_pending_writes(tx);
}
'''


def _ptxas(args, cwd):
    out = subprocess.run([NVCC] + ARCH + ["-O3", "-std=c++17", "-Xptxas", "-v"] + args, capture_output=True,
                         text=True, cwd=cwd)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stderr


def _kernels(report):
    """{kernel: (registers, spill stores, spill loads)} from a ptxas -v report"""
    res, name, spills = {}, None, (0, 0)
    for line in report.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            spills = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            res[name] = (int(m.group(1)),) + spills
    return res


def test_user_kernel_compiles_against_the_public_header():
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "user.cu"), "w") as f:
            f.write(USER_KERNEL)
        rep = _ptxas(["-I", os.path.join(ROOT, "include"), "-c", "user.cu", "-o", "user.o"], d)
        ks = _kernels(rep)
        assert any("echo" in k for k in ks), rep
        assert all(v[1] == 0 and v[2] == 0 for v in ks.values()), ks


def test_driver_compiles_for_sm90a_without_spills():
    with tempfile.TemporaryDirectory() as d:
        rep = _ptxas(["-Xcompiler", "-fPIC", "-shared", "-o", os.path.join(d, "libdevice_api.so"),
                      os.path.join(HERE, "native", "device_api.cu")], d)
        ks = _kernels(rep)
        assert any("da_kernel" in k for k in ks), rep
        for k, (regs, st, ld) in ks.items():
            assert st == 0 and ld == 0, (k, regs, st, ld)
        elf = subprocess.run(["cuobjdump", "-lelf", os.path.join(d, "libdevice_api.so")], capture_output=True,
                             text=True).stdout
        assert "sm_90a" in elf, elf


def test_handle_is_64_bytes_and_calls_are_exported(pkg):
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "h.c")
        with open(src, "w") as f:
            f.write('#include "b200_pair.h"\n_Static_assert(sizeof(b200_dev_pair) == 64, "size");\n'
                    'int main(void) { return 0; }\n')
        subprocess.check_call(["gcc", "-std=c11", "-Wall", "-I", os.path.join(ROOT, "include"), "-o",
                               os.path.join(d, "h"), src])
    L = pkg.lib()
    for s in ("b200_pair_device_claim", "b200_pair_device_release", "b200_pair_device_owned"):
        assert hasattr(L, s), s
        assert s in pkg.exported_symbols()
    assert pkg.DEV_PAIR_BYTES == 64
