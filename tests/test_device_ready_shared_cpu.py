"""CPU: an exhaustive check of a device ready set taken by several consumer warps at once (b200_warp_ready_take's
atomicCAS on the queue's head, DESIGN.md §13 "Many consumers"), extending the one-consumer model of
test_device_ready_cpu.py.

One member, one producer making one to three changes (a peer's Send, Recv or Disconnect: make the change, fence,
exchange `armed` with 0, and when it was 1 claim a position with atomicAdd(tail), then store the entry) and two or
three consumers.  A consumer takes
(load head, load the entry at that position -- a slot keeps its entry after it is taken, and an entry counts only at
the position its tag names -- then atomicCAS(head, h, h + 1), and on a lost CAS load head again), serves the member,
then rearms (store armed = 1, fence, probe, and on a ready probe exchange `armed` with 0 and keep the member if it was
1).  Both fences are modelled as sequentially consistent, so every interleaving of the single steps is a possible
execution.  A consumer holds the member from its won take or kept rearm until its rearm stores armed = 1; after that
store it only probes, which reads.  In every interleaving:
  - no change is left unreported once every side has nothing left to do (no lost wakeup);
  - the member never has more than one entry queued;
  - no two consumers hold the member at once.
The negative control takes with a plain store of head + 1 (the one-consumer take) and finds the member handed to two
consumers."""
import pytest

IDLE, READ, CAS, SERVE, STORE, PROBE, EXCH = range(7)
HOLDING = (SERVE, STORE)


def _explore(consumers, changes, initial_entry, cas_take=True):
    """Returns (max entries queued at once, lost wakeups, states where two consumers hold the member, states).
    State: (pp, left, ready, armed, head, tail, stored, cons); pp: producer step, stored: bitmask of positions whose
    entry has been stored, cons: per consumer (pc, h)."""
    start = (0, changes, False, 0 if initial_entry else 1, 0, 1 if initial_entry else 0, 1 if initial_entry else 0,
             ((IDLE, 0),) * consumers)
    seen, stack = set(), [start]
    max_q, lost, double = 0, 0, 0
    while stack:
        s = stack.pop()
        if s in seen:
            continue
        seen.add(s)
        pp, left, ready, armed, head, tail, stored, cons = s
        max_q = max(max_q, tail - head)
        if sum(1 for pc, _ in cons if pc in HOLDING) > 1:
            double += 1
        nxt = []
        # producer: 0 = make the change, 1 = (fence) exchange armed, 2 = claim a position, 3 = store the entry
        if left > 0:
            if pp == 0:
                nxt.append((1, left, True, armed, head, tail, stored, cons))
            elif pp == 1:
                if armed == 1:
                    nxt.append((2, left, ready, 0, head, tail, stored, cons))
                else:
                    nxt.append((0, left - 1, ready, armed, head, tail, stored, cons))
            elif pp == 2:
                nxt.append((3, left, ready, armed, head, tail + 1, stored, cons))
            else:  # the claimed position is tail - 1: a single producer claims one at a time
                nxt.append((0, left - 1, ready, armed, head, tail, stored | 1 << (tail - 1), cons))
        for c, (pc, h) in enumerate(cons):
            def put(npc, nh=h, **kw):
                st = dict(ready=ready, armed=armed, head=head)
                st.update(kw)
                nc = cons[:c] + ((npc, nh),) + cons[c + 1:]
                nxt.append((pp, left, st["ready"], st["armed"], st["head"], tail, stored, nc))
            if pc == IDLE:
                if tail != head:  # (an empty queue: the take returns 0 and the consumer polls again)
                    put(READ, head)
            elif pc == READ:  # load the entry at h: a run of one when its tag names h, else an empty take
                put(CAS if stored >> h & 1 else IDLE)
            elif pc == CAS:
                if head == h or not cas_take:
                    put(SERVE, head=h + 1)
                else:  # another consumer took first: load head again
                    put(READ, head)
            elif pc == SERVE:  # Recv until nothing is complete (everything), or stop early (the rest is still there)
                put(STORE, ready=False)
                put(STORE)
            elif pc == STORE:  # armed = 1, then the fence: the hold ends here, the probe only reads
                put(PROBE, armed=1)
            elif pc == PROBE:
                put(EXCH if ready else IDLE)
            elif pc == EXCH:
                put(SERVE if armed == 1 else IDLE, armed=0)
        if not nxt and ready:  # every side is done: a change nobody was told about is a lost wakeup
            lost += 1
        stack.extend(nxt)
    return max_q, lost, double, len(seen)


@pytest.mark.parametrize("initial_entry", [True, False], ids=["after-add", "armed"])
@pytest.mark.parametrize("changes", [1, 2, 3])
def test_two_consumers(changes, initial_entry):
    max_q, lost, double, states = _explore(2, changes, initial_entry)
    assert lost == 0
    assert max_q == 1
    assert double == 0
    assert states > 50


@pytest.mark.parametrize("initial_entry", [True, False], ids=["after-add", "armed"])
@pytest.mark.parametrize("changes", [1, 2, 3])
def test_three_consumers(changes, initial_entry):
    max_q, lost, double, states = _explore(3, changes, initial_entry)
    assert lost == 0 and max_q == 1 and double == 0
    assert states > 200


def test_one_consumer_as_before():
    # one consumer: the shared take is the one-consumer protocol with a CAS where the store was
    for changes in (1, 2, 3):
        for initial_entry in (True, False):
            assert _explore(1, changes, initial_entry)[:3] == (1, 0, 0)
            assert _explore(1, changes, initial_entry, cas_take=False)[:3] == (1, 0, 0)


def test_the_model_finds_a_key_handed_to_two_consumers_with_a_plain_store_take():
    # the one-consumer take (load head, load the entry, store head + 1) shared by two warps: both read the same
    # entry and both serve the member, so the check above has teeth
    _, _, double, _ = _explore(2, 1, True, cas_take=False)
    assert double > 0
