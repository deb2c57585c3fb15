"""CPU: the cluster kernels of B200_BATCH_CLUSTER (k_cluster_send / k_cluster_recv) are in the library, keep two CTAs
per SM without spills, and the flag needs no new C symbol; cluster_flag encodes the field.  No GPU needed."""
import subprocess

import pytest

import test_device_block_cpu as tb


def test_library_has_both_cluster_kernels(pkg):
    sass = subprocess.run(["cuobjdump", "-sass", pkg.LIB_PATH], capture_output=True, text=True).stdout
    for k in ("k_cluster_send", "k_cluster_recv"):
        assert "Function : _ZN4b200" in sass and k in sass, k
    # each one waits at cluster barriers
    parts = [p for p in sass.split("Function : ")[1:] if "k_cluster_" in p.split("\n", 1)[0]]
    assert len(parts) == 2 and all("UCGABAR_WAIT" in p for p in parts)


def test_cluster_kernels_fit_two_ctas_per_sm_without_spills():
    ks = tb._library_kernels()
    for name in ("k_cluster_send", "k_cluster_recv"):
        regs, st, ld, smem = tb._pick(ks, name)
        # __launch_bounds__(288, 2): at most 96 registers; the Recv kernel reads its op from shared memory and does
        # not spill (with the op in registers, as k_recv holds it, it spills 12 bytes)
        assert regs <= 96 and regs * 288 * 2 <= 65536, (name, regs)
        assert (st, ld) == (0, 0), (name, st, ld)
        assert 2 * (smem + tb.BLOCK_SMEM_BYTES + tb.SMEM_PER_CTA_RESERVED) <= tb.SMEM_PER_SM, (name, smem)
    # the kernels beside them keep their numbers
    assert tb._pick(ks, "k_send")[:3] == (80, 0, 0) and tb._pick(ks, "k_recv")[:3] == (96, 0, 0), ks
    assert tb._pick(ks, "k_svc_big")[:3] == (96, 20, 20), ks


def test_cluster_flag(pkg):
    assert [pkg.cluster_flag(k) for k in (1, 2, 4, 8, 16)] == [0x00, 0x10, 0x30, 0x70, 0xF0]
    for k in range(1, 17):
        f = pkg.cluster_flag(k)
        assert f & ~0xF0 == 0 and (f >> 4) + 1 == k
        # the other flags keep their bits
        assert f | pkg.UNTIL_BLOCKED | pkg.ZEROCOPY == f + 5
    for bad in (0, 17, -1, 32, 2.0, "2", None, True):
        with pytest.raises(ValueError):
            pkg.cluster_flag(bad)


def test_no_new_c_symbol(pkg):
    nm = subprocess.run(["nm", "-D", "--defined-only", pkg.LIB_PATH], capture_output=True, text=True, check=True)
    syms = {ln.split()[-1] for ln in nm.stdout.splitlines() if ln.split() and ln.split()[-1].startswith("b200_")}
    # the header's prototypes, which the binding table covers, and the service's debug hook
    assert syms == set(pkg._SIGS) | {"b200_debug_service_trace"}, sorted(syms ^ set(pkg._SIGS))
    assert not [s for s in pkg.exported_symbols() if "cluster" in s]
    hdr = open(pkg.HEADER).read()
    assert "#define B200_BATCH_CLUSTER(k) (((unsigned)(k) - 1u) << 4)" in hdr
