"""CPU model of the two-group schedule of lstm_layer_kernel (dorado_b200/csrc/lstm_model.cu, the fused LSTM layer of
lstm_size 96).  The kernel runs its 16 chunks as two groups, n tile 0 (chunks 0-7) and n tile 1 (chunks 8-15), half a step
apart, with one named barrier per group.  Its results are checked against the numpy oracle on the GPU
(tests/test_forward_gpu.py); this test pins the reasoning behind the schedule:
- a chunk's group is its n tile, and each group's ldmatrix fragments read only the group's rows of h and of the x ring;
- no h row or ring slot is overwritten before every warp has read it, every read sees the value of its step, and x_t is
  copied into the ring before h_t overwrites it in the sequence buffer.
The gate-row permutation and fragment ownership are modelled in tests/test_lstm_layer_logic_cpu.py."""
import pytest

C = 96               # FL_C
KS = C // 16         # FL_KS
HS = C + 8           # FL_HS
RING = 8             # FL_RING
AHEAD = RING - 1     # FL_AHEAD
WAIT = AHEAD - 2     # cp_async_wait<FL_AHEAD - 2>: copy groups that may stay in flight


def test_group_of_a_chunk_is_its_n_tile():
    # accumulators: the chunk of every (lane, n tile, element) lies in group n tile
    for lane in range(32):
        for nt in range(2):
            for el in range(4):
                chunk = 8 * nt + 2 * (lane % 4) + el % 2
                assert chunk // 8 == nt
    # B fragments: mma_group's ldmatrix.x4 at rows + kp * 64 bytes, lane address row qr, column qm * 8 (qm = lane / 8) of
    # the group's 8 rows.  Register j of lane l is row l / 4, columns 2 (l % 4) + {0, 1} of matrix j; the m16n8k16 B
    # fragment of k step ks is (k 2 (l % 4) + {0, 1}, + 8) x chunk l / 4.
    for group in range(2):
        rows = group * 8 * HS * 2   # FL_GROUP_BYTES
        for kp in range(KS // 2):
            addr = {}
            for lane in range(32):
                qm, qr = lane // 8, lane % 8
                addr[lane] = rows + (qr * HS + qm * 8) * 2 + kp * 64
            for lane in range(32):
                for j in range(4):
                    start = addr[8 * j + lane // 4] // 2 + 2 * (lane % 4)
                    chunk, k = divmod(start, HS)
                    ks = 2 * kp + j // 2
                    assert chunk == group * 8 + lane // 4
                    assert k == ks * 16 + 8 * (j % 2) + 2 * (lane % 4)
                    assert k + 1 < C


def layer_schedule(T, ahead=AHEAD, wait=WAIT, prologue_barrier=True):
    """The shared-memory and sequence-buffer accesses of lstm_layer_kernel in program order, as (phase, op, args).  A phase
    is the interval between two CTA barriers; accesses of different warps in one phase are unordered.  Ops: copy (cp.async
    of x(step) issued), done (the copies of steps <= n complete in every thread before the barrier that ends the phase),
    read_x (step, group), read_h / write_h (group, step), write_seq (group, step).  h is one buffer per group."""
    ops, phase = [], 0
    committed = 0

    def copy(step):
        nonlocal committed
        ops.append((phase, "copy", step))
        committed += 1

    for s in range(ahead):
        copy(s)
    for g in range(2):
        ops.append((phase, "write_h", g, -1))
    ops.append((phase, "done", committed - wait - 1))
    phase += 1                                          # __syncthreads
    ops += [(phase, "read_x", 0, 0), (phase, "read_x", 0, 1), (phase, "read_h", 0, -1)]
    phase += prologue_barrier                           # __syncthreads
    for s in range(T):
        ops.append((phase, "read_h", 1, s - 1))            # W_hh h_B(s-1)
        ops += [(phase, "write_h", 0, s), (phase, "write_seq", 0, s)]
        ops.append((phase, "read_x", s + 1, 0))                          # W_ih x_A(s+1)
        phase += 1                                                       # barrier A
        ops.append((phase, "read_h", 0, s))                      # W_hh h_A(s)
        ops += [(phase, "write_h", 1, s), (phase, "write_seq", 1, s)]
        ops.append((phase, "read_x", s + 1, 1))                          # W_ih x_B(s+1)
        copy(s + ahead)
        ops.append((phase, "done", committed - wait - 1))
        phase += 1                                                       # barrier B
    return ops


def schedule_violations(T, **kw):
    ops = layer_schedule(T, **kw)
    found = []
    # h: a read sees the write of its step from an earlier phase, and no warp writes the group's rows in the read's phase
    writes = [(p, g, step) for p, op, *a in ops if op == "write_h" for g, step in [a]]
    for p, op, *a in ops:
        if op != "read_h":
            continue
        g, step = a
        before = [(wp, ws) for wp, wg, ws in writes if wg == g and wp < p]
        if not before or max(before)[1] != step:
            found.append(("h read sees another step", g, step))
        if any(wp == p for wp, wg, ws in writes if wg == g):
            found.append(("h written in the phase of a read", g, step))
    # ring: x(j) is visible from the phase after the barrier whose `done` covers it; the next copy into its slot is issued
    # in a later phase than every read of x(j).  Products of step T and later are never read.
    issued = {a[0]: p for p, op, *a in ops if op == "copy"}
    visible = {}
    for p, op, *a in ops:
        if op == "done":
            for j in range(a[0] + 1):
                visible.setdefault(j, p + 1)
    for p, op, *a in ops:
        if op == "read_x" and a[0] < T:
            j = a[0]
            if visible.get(j, 1 << 30) > p:
                found.append(("x read before its copy is visible", j))
            if j + RING in issued and issued[j + RING] <= p:
                found.append(("ring slot overwritten before a read", j))
        if op == "write_seq" and visible.get(a[1], 1 << 30) > p:
            found.append(("h written over x before its copy completed", a[1]))
    return found


@pytest.mark.parametrize("T", [1, 2, 3, 7, 8, 9, 40, 1666])
def test_staggered_schedule_has_no_hazard(T):
    assert schedule_violations(T) == []


def test_schedule_model_finds_hazards():
    # the checks are not vacuous: one more step of prefetch reuses a slot still being read, one fewer wait publishes x
    # too late, and without the barrier after the prologue step 0 writes h_A(0) while a warp may still read h_A(-1)
    assert ("ring slot overwritten before a read", 1) in schedule_violations(40, ahead=RING + 1)
    assert ("x read before its copy is visible", 2) in schedule_violations(40, wait=WAIT + 1)
    assert schedule_violations(40, prologue_barrier=False) == [("h written in the phase of a read", 0, -1)]
