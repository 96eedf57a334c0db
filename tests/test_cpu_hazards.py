"""CPU tier: hazard check of the fused MLP program's overlapped schedule (Builder::finalize in csrc/pnr_api.cu).
The sm_90 kernel does not execute this schedule (it runs a step's epilogue after all of the step's MMAs; see
"UNUSED ON SM_90" in csrc/mlp_program.h); the test pins that the program's flags stay self-consistent.

The program keeps accumulators, activations (16-bit hi / lo parts) and head activations in overlapping operand-column
ranges and orders the MMA stages against the epilogue parts of every step with
  * MMA commit -> mbarrier:  acc_full[0/1] (F_COMMIT_ACC0/1), war_ok (F_COMMIT_WAR),
  * three monotonic counters epilogue -> MMA issuer (E0 done, E1 part a done, E1 done): every stage of the issue
    table carries the counts it needs (IssueDesc.needs).
Their placement is computed on the host.  This test rebuilds the happens-before graph they imply, over two
consecutive tiles, and requires that every pair of events that touch overlapping columns with at least one write
is ordered by it."""
import itertools

import pytest

from panopticnerf_b200 import make_cfg, make_network, synthetic as S
from test_cpu_program import (A_TMEM, EPI_LOADG_TO_A, EPI_MASK_TO_A, EPI_RELU_TO_A, F_COMMIT_ACC0, F_COMMIT_ACC1,
                              F_COMMIT_VIEW, F_COMMIT_WAR, F_WAIT_E0, F_WAIT_E1, F_WAIT_E1A, PROGRAM_BACKWARD,
                              PROGRAM_NO_SPLIT, PROGRAM_SPLIT_E1, PROGRAM_VIEW_PRODUCERS, build)


def overlap(a, b):
    return a[0] < a[1] and b[0] < b[1] and a[0] < b[1] and b[0] < a[1]


def events_and_edges(prog, tiles=3):
    """Events of step s of tile t (aggregated over the epilogue warps):
      ('S', t, i)    MMA stage i
      ('L0', t, s)   E0's accumulator loads            (after acc_full[0])
      ('W0', t, s)   E0's stores                         (after war_ok)
      ('E1a', t, s) / ('E1b', t, s) E1's loads + stores, part a / b (after acc_full[1])
      ('D0', t, s), ('D1a', t, s), ('D1', t, s)   the three hand-off counters reaching this step's count
      ('EV', t), ('DV', t)   view-on-producers programs: the view epilogue of tile t on the producer warps (after the
                             view step's own commit) and its counter; that step has no E0 / E1 events
    Returns (reads, writes, edges)."""
    x3 = prog.passes == 3
    steps = []
    for i in range(prog.n_stages):
        if prog.st[i].flags & F_WAIT_E0:
            steps.append([])
        steps[-1].append(i)
    n_steps = len(steps)
    vs = prog.view_step                                  # -1, or the (last) step the producer warps finish
    n_esteps = n_steps - 1 if vs >= 0 else n_steps       # steps in the E0 / E1 counts
    reads, writes, edges = {}, {}, []
    order = [(t, s) for t in range(tiles) for s in range(n_esteps)]     # what the epilogue warps run, in their order
    gidx = {ts: k for k, ts in enumerate(order)}

    def fl(t, a0, a1):
        """accumulator interval of tile t: odd tiles use the columns XOR 128 when the program flips (no range straddles 128)"""
        if prog.acc_flip and (t & 1) and a0 < a1:
            assert a0 // 128 == (a1 - 1) // 128
            return (a0 ^ 128, (a0 ^ 128) + (a1 - a0))
        return (a0, a1)

    def cols(t, ed, c0, c1, to_a):
        """(accumulator interval read, activation intervals written) of epilogue columns [c0, c1) in tile t."""
        r = [fl(t, ed.acc_col + c0, ed.acc_col + c1)] if c0 < c1 else []
        w = []
        if to_a and c0 < c1:
            w = [(ed.dst_col + c0 // 2, ed.dst_col + c1 // 2)] + (
                [(ed.dst_lo_col + c0 // 2, ed.dst_lo_col + c1 // 2)] if x3 else [])
        return r, w

    prev_stage = None
    for t, s in [(t, s) for t in range(tiles) for s in range(n_steps)]:
        ed = prog.ep[s]
        to_a = ed.kind in (EPI_RELU_TO_A, EPI_MASK_TO_A, EPI_LOADG_TO_A)
        for i in steps[s]:
            sd = prog.st[i]
            ev = ("S", t, i)
            r = [fl(t, sd.acc_col, sd.acc_col + sd.n)]
            if sd.a_kind == A_TMEM:
                r.append((sd.a_off, sd.a_off + 8 * sd.ksteps))
                if x3:
                    r.append((sd.a_lo_off, sd.a_lo_off + 8 * sd.ksteps))
            reads[ev], writes[ev] = r, [fl(t, sd.acc_col, sd.acc_col + sd.n)]
            if prev_stage is not None:
                edges.append((prev_stage, ev))        # the tensor pipe retires MMAs in issue order
            prev_stage = ev
            if sd.flags & F_COMMIT_ACC0:     # a warp stores only after it has passed acc_full[0] itself
                edges += [(ev, ("L0", t, s)), (ev, ("W0", t, s))]
            if sd.flags & F_COMMIT_ACC1:
                edges += [(ev, ("E1a", t, s)), (ev, ("E1b", t, s))]
            if sd.flags & F_COMMIT_WAR:
                edges.append((ev, ("W0", t, s)))
            if sd.flags & F_COMMIT_VIEW:
                edges.append((ev, ("EV", t)))
            if (prog.is_[i].needs >> 24) and t >= 1:
                edges.append((("DV", t - 1), ev))
            # hand-off counts: v - 1 steps of this tile (and all earlier tiles) have completed that part
            needs = prog.is_[i].needs
            for shift, name in ((0, "D0"), (8, "D1a"), (16, "D1")):
                g = t * n_esteps + ((needs >> shift) & 0xFF) - 2      # global index of the last step required
                if g >= 0:
                    edges.append(((name,) + order[g], ev))
        if s == vs:      # the producer warps read the whole accumulator of the step and write no operand column
            reads[("EV", t)], writes[("EV", t)] = cols(t, ed, 0, ed.n, False)[0], []
            reads[("DV", t)], writes[("DV", t)] = [], []
            edges.append((("EV", t), ("DV", t)))
            if t >= 1:
                edges.append((("DV", t - 1), ("DV", t)))      # each producer warp runs the tiles in order
            continue
        # a step issued as one half signals acc_full[0] and [1] from its last stage
        if not any(prog.st[i].flags & F_COMMIT_ACC0 for i in steps[s]):
            edges += [(("S", t, steps[s][-1]), (e, t, s)) for e in ("L0", "W0")]
        reads[("L0", t, s)], writes[("L0", t, s)] = cols(t, ed, 0, ed.n0, False)[0], []
        reads[("W0", t, s)], writes[("W0", t, s)] = [], cols(t, ed, 0, ed.n0, to_a)[1]
        reads[("E1a", t, s)], writes[("E1a", t, s)] = cols(t, ed, ed.n0, ed.n1a, to_a)
        reads[("E1b", t, s)], writes[("E1b", t, s)] = cols(t, ed, ed.n1a, ed.n, to_a)
        for d in ("D0", "D1a", "D1"):
            reads[(d, t, s)], writes[(d, t, s)] = [], []
        edges += [(("L0", t, s), ("D0", t, s)), (("W0", t, s), ("D0", t, s)),
                  (("E1a", t, s), ("D1a", t, s)), (("E1b", t, s), ("D1", t, s)),
                  # every warp bumps its counters in program order, so a count implies the earlier ones
                  (("D0", t, s), ("D1a", t, s)), (("D1a", t, s), ("D1", t, s))]
        if gidx[(t, s)] + 1 < len(order):
            edges.append((("D1", t, s), ("D0",) + order[gidx[(t, s)] + 1]))
    return reads, writes, edges


def reachability(nodes, edges):
    idx = {n: k for k, n in enumerate(nodes)}
    succ = [[] for _ in nodes]
    for a, b in edges:
        succ[idx[a]].append(idx[b])
    reach = []
    for k in range(len(nodes)):
        seen, stack = set(), [k]
        while stack:
            v = stack.pop()
            for w in succ[v]:
                if w not in seen:
                    seen.add(w)
                    stack.append(w)
        reach.append(seen)
    return idx, reach


def unordered_conflicts(prog):
    reads, writes, edges = events_and_edges(prog)
    nodes = list(reads)
    idx, reach = reachability(nodes, edges)
    checked, bad = 0, []
    for a, b in itertools.combinations(nodes, 2):
        if a[0] == "S" and b[0] == "S":
            continue                                    # MMAs are ordered among themselves by construction
        conflict = any(overlap(x, y) for x in writes[a] for y in reads[b] + writes[b]) or \
                   any(overlap(x, y) for x in writes[b] for y in reads[a])
        if not conflict:
            continue
        checked += 1
        if not (idx[b] in reach[idx[a]] or idx[a] in reach[idx[b]]):
            bad.append((a, b))
    return checked, bad


CASES = [("cfg1", {}), ("cfg2", {}), ("cfg3", {}), ("cfg2", dict(precision="fp16")),
         ("cfg2", dict(D=5, W=128, num_classes=7, num_instances=3)), ("cfg3", dict(precision="bf16x3", W=128)),
         ("cfg1", dict(D=3, num_classes=45))]


@pytest.mark.parametrize("preset,over", CASES)
@pytest.mark.parametrize("flags", [0, PROGRAM_NO_SPLIT, PROGRAM_SPLIT_E1])
def test_every_tensor_memory_conflict_is_ordered(preset, over, flags):
    """Default program of the precision, one-block E1, two-block E1."""
    cfg = make_cfg(preset, **over)
    prog, _, _ = build(cfg, S.init_network_weights(make_network(cfg), seed=0), flags=flags)
    checked, bad = unordered_conflicts(prog)
    assert checked > 20
    assert not bad, f"{preset} {over} flags={flags}: unordered tensor-memory conflicts, e.g. {bad[:3]}"


@pytest.mark.parametrize("preset,over", [("cfg2", {}), ("cfg2", dict(precision="bf16x3", D=5, W=128)), ("cfg1", dict(D=3, W=64))])
@pytest.mark.parametrize("flags", [0, PROGRAM_NO_SPLIT])
def test_backward_program_conflicts_are_ordered(preset, over, flags):
    """The backward program of the trunk (forward steps + the layers in reverse) under the same analysis."""
    cfg = make_cfg(preset, **over)
    prog, _, _ = build(cfg, S.init_network_weights(make_network(cfg), seed=0), flags=flags | PROGRAM_BACKWARD)
    checked, bad = unordered_conflicts(prog)
    assert checked > 20
    assert not bad, f"{preset} {over} flags={flags}: unordered tensor-memory conflicts, e.g. {bad[:3]}"


@pytest.mark.parametrize("preset,over", [("cfg2", {}), ("cfg2", dict(precision="fp16")), ("cfg1", {}), ("cfg1", dict(D=3, W=128, xyz_res=4)),
                                         ("cfg2", dict(precision="bf16x3", D=5, W=128))])
@pytest.mark.parametrize("flags", [0, PROGRAM_NO_SPLIT])
def test_view_on_producers_conflicts_are_ordered(preset, over, flags):
    """The variant whose view epilogue runs on the producer warps (own commit barrier, own counter) under the same
    analysis; and dropping the gate on the producer counter is noticed."""
    cfg = make_cfg(preset, **over)
    prog, _, _ = build(cfg, S.init_network_weights(make_network(cfg), seed=0), flags=flags | PROGRAM_VIEW_PRODUCERS)
    assert prog.view_step == prog.n_steps - 1
    checked, bad = unordered_conflicts(prog)
    assert checked > 20
    assert not bad, f"{preset} {over} flags={flags}: unordered tensor-memory conflicts, e.g. {bad[:3]}"
    for i in range(prog.n_stages):
        prog.is_[i].needs &= 0x00FFFFFF
    _, bad = unordered_conflicts(prog)
    assert bad


@pytest.mark.parametrize("preset,over", [("cfg2", {}), ("cfg3", {}), ("cfg2", dict(D=5, W=128, num_classes=7, num_instances=3))])
def test_split_e1_waits_later_for_the_second_block(preset, over):
    """With E1 in two blocks, the wait on part a comes no later than the wait on all of E1, and the latter moves
    later wherever a half spans several weight stages (that is the point: the third K-chunk starts earlier)."""
    cfg = make_cfg(preset, **over)
    net = S.init_network_weights(make_network(cfg), seed=0)
    prog, _, _ = build(cfg, net, flags=PROGRAM_SPLIT_E1)
    base, _, _ = build(cfg, net, flags=PROGRAM_NO_SPLIT)
    assert prog.n_stages == base.n_stages

    def where(p, flag):
        return [i for i in range(p.n_stages) if p.st[i].flags & flag]
    assert where(prog, F_COMMIT_WAR) == where(base, F_COMMIT_WAR) and len(where(prog, F_COMMIT_WAR)) == prog.n_steps
    assert where(base, F_WAIT_E1A) == where(base, F_WAIT_E1)
    e1a, e1, e1_base = where(prog, F_WAIT_E1A), where(prog, F_WAIT_E1), where(base, F_WAIT_E1)
    assert all(a <= b for a, b in zip(e1a, e1)) and all(b >= c for b, c in zip(e1, e1_base))
    if cfg.W >= 256:     # a 256-wide x3 layer has 4 weight stages per half
        assert any(b > c for b, c in zip(e1, e1_base))


def test_the_checker_sees_a_missing_wait():
    """Drop one stage's wait on E1 and the same analysis must find an unordered conflict (the check is not vacuous)."""
    cfg = make_cfg("cfg2")
    prog, _, _ = build(cfg, S.init_network_weights(make_network(cfg), seed=0))
    # a stage inside a trunk layer (the tile's first step follows a step whose second epilogue part may be empty)
    first_of_step1 = [i for i in range(prog.n_stages) if prog.st[i].flags & F_WAIT_E0][1]
    victim = next(i for i in range(first_of_step1, prog.n_stages)
                  if prog.st[i].flags & F_WAIT_E1 and not prog.st[i].flags & F_WAIT_E0)
    needs = prog.is_[victim].needs
    prog.is_[victim].needs = (needs & 0xFF00FFFF) | ((((needs >> 16) & 0xFF) - 1) << 16)
    _, bad = unordered_conflicts(prog)
    assert bad
