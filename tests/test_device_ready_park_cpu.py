"""CPU: parking a device ready set (DESIGN.md §13 "Parking"): the control words' layout, compiled for the host, and an
exhaustive check of the park / push / ring protocol.

The model runs one member and one to three producers.  Each makes one change (a peer's Send, Recv or Disconnect):
make the change, fence, exchange `armed` with 0, and when it was 1 claim a position with the 64-bit atomicAdd on the
tail word, store the entry, and when the add returned the parked bit, clear it with atomicAnd and ring when the And
still saw it.  The consumer is a server that the host launches when it sees a ring it has not answered: take, serve,
rearm (store armed = 1, fence, probe, exchange on a ready probe), and on an empty take park (atomicOr of the bit,
compare the tail it covered with head; not equal: atomicAnd, and non-zero when the bit was still set).  On 0 it exits;
on non-zero it takes again.  The host park is the same park with no server running, before any server was launched.
The fences are sequentially consistent and park and push are read-modify-writes of one word, so every interleaving of
the single steps is a possible execution.  In every one:
  - a park that returned 0 is answered by exactly one ring, or by none when no change came after it;
  - a park that returned non-zero leaves entries queued, which the server then takes;
  - no change is left unreported with the set parked, the queue non-empty and no ring (no lost wakeup);
  - never two rings for one park.
Negative controls: a park that stores the bit and reads the tail separately with no fence between them (the read
goes first), and a push that reads the bit before its add.  The model finds the lost wakeup in each."""
import ctypes as C
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")

# consumer states
OFF, TAKE, SERVE, STORE, PROBE, EXCH, PARK, PARK_AND, HOSTPARK, SPLIT_READ, SPLIT_CMP = range(11)


def _explore(producers, initial_entry, host_park, split_park=False, read_bit_first=False):
    """Returns dict of counts over all reachable states.  State: (prods, ready, armed, head, tail, stored, parked,
    rings, parks0, answered, cons, low); prods: per producer (step, pos, bit)."""
    start_cons = HOSTPARK if host_park else TAKE
    start = (((0, 0, 0),) * producers, False, 0 if initial_entry else 1, 0, 1 if initial_entry else 0,
             1 if initial_entry else 0, 0, 0, 0, 0, start_cons, 0)
    seen, stack = set(), [start]
    res = dict(states=0, lost=0, double_ring=0, busy_empty=0, unanswered_bad=0, terminals=0, max_q=0)
    while stack:
        s = stack.pop()
        if s in seen:
            continue
        seen.add(s)
        prods, ready, armed, head, tail, stored, parked, rings, parks0, answered, cons, low = s
        res["max_q"] = max(res["max_q"], tail - head)
        if rings > parks0:
            res["double_ring"] += 1
        nxt = []

        def put(**kw):
            st = dict(prods=prods, ready=ready, armed=armed, head=head, tail=tail, stored=stored, parked=parked,
                      rings=rings, parks0=parks0, answered=answered, cons=cons, low=low)
            st.update(kw)
            nxt.append((st["prods"], st["ready"], st["armed"], st["head"], st["tail"], st["stored"], st["parked"],
                        st["rings"], st["parks0"], st["answered"], st["cons"], st["low"]))

        DONE = 9
        for i, (step, pos, bit) in enumerate(prods):
            def pset(nstep, npos=pos, nbit=bit, **kw):
                put(prods=prods[:i] + ((nstep, npos, nbit),) + prods[i + 1:], **kw)
            if step == 0:  # the change
                pset(1, ready=True)
            elif step == 1:  # fence, exchange armed
                if armed == 1:
                    pset(7 if read_bit_first else 2, armed=0)
                else:
                    pset(DONE)
            elif step == 7:  # negative control: read the bit, then add
                pset(8, nbit=parked)
            elif step == 8:
                pset(3, npos=tail, tail=tail + 1)
            elif step == 2:  # 64-bit atomicAdd: the position and the parked bit in one
                pset(3, npos=tail, nbit=parked, tail=tail + 1)
            elif step == 3:  # store the entry
                pset(4 if bit else DONE, stored=stored | 1 << pos)
            elif step == 4:  # atomicAnd: the one that still saw the bit rings
                pset(5 if parked else DONE, parked=0)
            elif step == 5:  # fence, store the ring count
                pset(DONE, rings=rings + 1)

        if cons == OFF:
            if rings > answered:  # the host saw the fd, consumes it and launches a server
                put(cons=TAKE, answered=rings)
        elif cons == TAKE:
            if tail != head and stored >> head & 1:
                put(cons=SERVE, head=head + 1)
            else:
                put(cons=SPLIT_READ if split_park else PARK)
        elif cons == SERVE:  # Recv until nothing is complete (everything), or stop early
            put(cons=STORE, ready=False)
            put(cons=STORE)
        elif cons == STORE:
            put(cons=PROBE, armed=1)
        elif cons == PROBE:
            put(cons=EXCH if ready else TAKE)
        elif cons == EXCH:
            put(cons=SERVE if armed == 1 else TAKE, armed=0)
        elif cons in (PARK, HOSTPARK):  # atomicOr(bit): the covered tail against head
            if tail == head:
                put(cons=OFF, parked=1, parks0=parks0 + 1)
            else:
                put(cons=PARK_AND, parked=1)
        elif cons == PARK_AND:
            if parked:  # nobody rang: entries are queued, serve them
                if tail == head:
                    res["busy_empty"] += 1
                put(cons=TAKE, parked=0)
            else:  # a producer cleared the bit: its ring is on its way
                put(cons=OFF, parks0=parks0 + 1)
        elif cons == SPLIT_READ:  # negative control: the tail read went before the store of the bit
            put(cons=SPLIT_CMP, low=tail)
        elif cons == SPLIT_CMP:  # the store of the bit, then the compare of what was read
            if low == head:
                put(cons=OFF, parked=1, parks0=parks0 + 1)
            else:
                put(cons=TAKE)
        if not nxt:
            res["terminals"] += 1
            pending = ready or tail != head
            if pending:
                res["lost"] += 1
            # every park that returned 0 but the last was answered by a ring; the last one too, unless nothing came
            if not (rings == parks0 or (rings == parks0 - 1 and parked and tail == head)):
                res["unanswered_bad"] += 1
        stack.extend(nxt)
    res["states"] = len(seen)
    return res


CASES = [(p, init, host) for p in (1, 2, 3) for init in (True, False) for host in (False, True)]


@pytest.mark.parametrize("producers,initial_entry,host_park", CASES)
def test_park_protocol(producers, initial_entry, host_park):
    r = _explore(producers, initial_entry, host_park)
    assert r["lost"] == 0, r
    assert r["double_ring"] == 0, r
    assert r["busy_empty"] == 0, r
    assert r["unanswered_bad"] == 0, r
    assert r["max_q"] <= 1, r
    assert r["states"] > 20 and r["terminals"] > 0, r


@pytest.mark.parametrize("producers", [1, 2])
def test_negative_control_split_park(producers):
    # the bit stored and the tail read as two operations, the read first: a push between them sees no bit, and the
    # park sees an empty queue -- the entry stays queued on a parked set with no ring
    r = _explore(producers, False, False, split_park=True)
    assert r["lost"] > 0


@pytest.mark.parametrize("producers", [1, 2])
def test_negative_control_bit_read_before_add(producers):
    # a push that reads the parked bit and then adds: a park between the two is never answered
    r = _explore(producers, False, False, read_bit_first=True)
    assert r["lost"] > 0


@pytest.fixture(scope="module")
def pa():
    subprocess.check_call(["make", "-s", "-C", NATIVE, "-f", "device_ready_park.mk", "park_arith.so"])
    L = C.CDLL(os.path.join(NATIVE, "park_arith.so"))
    for f in ("pa_sizeof_queue", "pa_offset_head", "pa_offset_tail", "pa_offset_tail_hi", "pa_offset_rings",
              "pa_offset_mask", "pa_offset_bell", "pa_entries_offset", "pa_parked_bit"):
        getattr(L, f).restype = C.c_uint64
    return L


def test_layout(pa):
    # the 384-byte layout of test_device_ready_cpu.py holds; the new words live in the padding of its lines
    assert pa.pa_sizeof_queue() == 384 and pa.pa_entries_offset() == 384
    assert pa.pa_offset_head() == 0 and pa.pa_offset_tail() == 128 and pa.pa_offset_mask() == 256
    # the parked bit is bit 63 of the 64-bit word at 128, whose low half is tail
    assert pa.pa_offset_tail_hi() == 132 and pa.pa_parked_bit() == 1 << 63
    assert 136 <= pa.pa_offset_rings() and pa.pa_offset_rings() + 8 <= 256
    assert 260 <= pa.pa_offset_bell() and pa.pa_offset_bell() + 8 <= 384 and pa.pa_offset_bell() % 8 == 0


def test_binding_and_symbols(pkg):
    for name in ("b200_ready_set_park", "b200_ready_set_wakeup_fd", "b200_ready_set_consume_wakeup",
                 "b200_ready_set_rings"):
        assert name in pkg.exported_symbols() and name in pkg._SIGS
    for meth in ("park", "wakeup_fd", "consume_wakeup", "rings"):
        assert callable(getattr(pkg.ReadySet, meth))
    dev = open(os.path.join(HERE, "..", "include", "b200_device.cuh")).read()
    assert "b200_warp_ready_park(const b200_dev_ready_set* s)" in dev
