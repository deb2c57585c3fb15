"""CPU: the device ready sets' queue arithmetic (the B200_HD inlines of csrc/b200_dev.cuh, compiled here for the host)
and an exhaustive check of the armed / entry protocol of notify_peer and b200_warp_ready_take / rearm.

The protocol model runs one producer (a peer's Send, Recv or Disconnect: make the change, then exchange `armed` with 0
and append the key if it was 1) against the one consumer (take an entry, serve, then rearm: store armed = 1, probe,
and on a ready probe exchange `armed` with 0 and keep the end if it was 1).  Both fences are modelled as sequentially
consistent, so every interleaving of the single steps is a possible execution.  In every one of them a member never
has two entries queued, and once both sides have nothing left to do no change is left unreported."""
import ctypes as C
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")


@pytest.fixture(scope="module")
def ra():
    subprocess.check_call(["make", "-s", "-C", NATIVE, "-f", "device_ready.mk", "ready_arith.so"])
    L = C.CDLL(os.path.join(NATIVE, "ready_arith.so"))
    u32, u64 = C.c_uint32, C.c_uint64
    L.ra_queue_size.restype, L.ra_queue_size.argtypes = u32, [u32]
    L.ra_add_check.restype, L.ra_add_check.argtypes = C.c_int, [u32] * 5
    L.ra_entry.restype, L.ra_entry.argtypes = u64, [u32, u32]
    L.ra_entry_at.restype, L.ra_entry_at.argtypes = C.c_int, [u64, u32]
    L.ra_note_offset.restype, L.ra_note_offset.argtypes = u64, [C.c_int]
    for f in ("ra_sizeof_queue", "ra_sizeof_note", "ra_offset_tail", "ra_offset_mask", "ra_entries_offset"):
        getattr(L, f).restype = u64
    return L


def test_layouts(ra):
    # head, tail and the read-only mask on three separate 128-byte lines, the entries after them
    assert ra.ra_sizeof_queue() == 384 and ra.ra_offset_tail() == 128 and ra.ra_offset_mask() == 256
    assert ra.ra_entries_offset() == 384
    # the notes follow the 8192 PairDev rows (128 B) and the 8192 PairSeq (16 B) of the connection table
    assert ra.ra_sizeof_note() == 16
    assert ra.ra_note_offset(0) == 8192 * (128 + 16)
    assert ra.ra_note_offset(8191) == 8192 * (128 + 16) + 16 * 8191


def test_queue_size(ra):
    for cap in (1, 2, 3, 4, 5, 31, 32, 33, 1000, 1024, 4096, 8191, 8192):
        s = ra.ra_queue_size(cap)
        assert s & (s - 1) == 0 and s >= 2 * cap and s < 4 * cap, (cap, s)


def test_entries_and_wrap(ra):
    for pos in (0, 1, 4095, 4096, 0x7FFFFFFF, 0xFFFFFFFE, 0xFFFFFFFF):
        for key in (0, 1, 0xDEADBEEF, 0xFFFFFFFF):
            e = ra.ra_entry(key, pos)
            assert e & 0xFFFFFFFF == key
            assert ra.ra_entry_at(e, pos) == 1
            assert ra.ra_entry_at(e, (pos + 1) & 0xFFFFFFFF) == 0
            assert ra.ra_entry_at(e, (pos - 1) & 0xFFFFFFFF) == 0
        # a slot never written reads as 0: no position before the stream wraps matches it
        if pos != 0xFFFFFFFF:
            assert ra.ra_entry_at(0, pos) == 0
    # the slot of a position one lap earlier never passes for the current one
    size = 8
    for pos in range(size, 3 * size):
        assert ra.ra_entry_at(ra.ra_entry(7, pos - size), pos) == 0


def test_add_check(ra):
    OK, FULL, OVERFLOW = 0, 1, 2
    cap = 4
    size = ra.ra_queue_size(cap)  # 8
    # no stale entries: a set that is not full always takes one more member
    for members in range(cap):
        for queued in range(members + 1):
            for head in (0, 5, 0xFFFFFFFF - 2):
                tail = (head + queued) & 0xFFFFFFFF
                assert ra.ra_add_check(head, tail, members, cap, size) == OK
    assert ra.ra_add_check(0, 0, cap, cap, size) == FULL
    # stale entries of released members count until they are taken
    assert ra.ra_add_check(0, 5, 3, cap, size) == OVERFLOW
    assert ra.ra_add_check(0, 4, 3, cap, size) == OK
    assert ra.ra_add_check(0xFFFFFFFE, 3, 2, cap, size) == OK        # 5 queued across the wrap of the stream
    assert ra.ra_add_check(0xFFFFFFFE, 4, 2, cap, size) == OVERFLOW  # 6 queued + 2 members


# ---- the protocol, exhaustively

def _explore(changes, initial_entry, rearm_probes=True):
    """All interleavings of a producer making `changes` readiness changes and the consumer.  Returns (max entries
    queued at once, lost wakeups found, states visited).  State: (pc_p, pc_c, ready, armed, queued, left)."""
    start = (0, "idle", False, 0 if initial_entry else 1, 1 if initial_entry else 0, changes)
    seen, stack = set(), [start]
    max_q, lost = 0, 0
    while stack:
        s = stack.pop()
        if s in seen:
            continue
        seen.add(s)
        pp, pc, ready, armed, q, left = s
        max_q = max(max_q, q)
        nxt = []
        # producer: 0 = make the change, 1 = (fence) exchange armed, 2 = append
        if left > 0:
            if pp == 0:
                nxt.append((1, pc, True, armed, q, left))
            elif pp == 1:
                nxt.append((2 if armed == 1 else 0, pc, ready, 0, q, left if armed == 1 else left - 1))
            elif pp == 2:
                nxt.append((0, pc, ready, armed, q + 1, left - 1))
        # consumer
        if pc == "idle":
            if q > 0:
                nxt.append((pp, "serve", ready, armed, q - 1, left))
        elif pc == "serve":  # Recv until nothing is complete (everything), or stop early (the rest is still there)
            nxt.append((pp, "store", False, armed, q, left))
            nxt.append((pp, "store", ready, armed, q, left))
        elif pc == "store":  # armed = 1, then the fence
            nxt.append((pp, "probe" if rearm_probes else "idle", ready, 1, q, left))
        elif pc == "probe":
            nxt.append((pp, "exch" if ready else "idle", ready, armed, q, left))
        elif pc == "exch":
            nxt.append((pp, "serve" if armed == 1 else "idle", ready, 0, q, left))
        if not nxt:  # both sides are done: a change nobody was told about is a lost wakeup
            if ready:
                lost += 1
        stack.extend(nxt)
    return max_q, lost, len(seen)


@pytest.mark.parametrize("initial_entry", [True, False], ids=["after-add", "armed"])
@pytest.mark.parametrize("changes", [1, 2, 3])
def test_no_lost_wakeup_and_one_entry(changes, initial_entry):
    max_q, lost, states = _explore(changes, initial_entry)
    assert lost == 0
    assert max_q == 1
    assert states > 10


def test_the_model_finds_a_lost_wakeup_without_the_probe():
    # a rearm that only stores armed = 1 loses the change that raced with it: the check above has teeth
    _, lost, _ = _explore(2, True, rearm_probes=False)
    assert lost > 0
