"""The evaluation kernels (pnr_eval_semantic / pnr_eval_panoptic / pnr_eval_image) at the limits they accept, through
lib/evaluators/ops.py, against oracle/reference_eval.py or against tallies known by construction where the oracle's
per-pair loop is too slow.  Counts are exact and iou_sum is bit-equal to math.fsum of the frame's IoUs.

- The 128-bit IoU accumulator: one channel with 2047 .. 2^17 + 3 matches (an id table maps hundreds of dataset ids to
  it), so the 64-bit low word wraps once or many times; exact ties of the final rounding and one unit either side.
- The integer decision boundaries on the device: every closed-form frame of test_cpu_eval.py, 2 inter == union
  against 2 inter == union + 1, and 2 ignored == area against 2 ignored == area + 1 (void, crowd and both).
- The open-addressing tables: all-distinct pairs filling them to exactly half, and keys whose home slot is among the
  last 8 of each table, so that probe chains of hundreds of slots wrap from slot S - 1 to 0.
- Id edges: INT32_MAX / INT32_MIN / negative ids / id 0, the first and last dataset id of every table, table entries
  -1 / C - 1 / C, and a 2 147 484-entry table that maps INT32_MAX.
- Size: a panoptic frame of 2^24 pixels (its workspace is 44 x 2^25 bytes + 13 KB; pnr_eval_panoptic near 2^31
  pixels would need ~190 GB of workspace, so 2^24 is its largest size tested), a semantic frame of 2^31 - 1 pixels
  (one 8 GiB buffer, skipped when the device has less free memory) and the refusal of 2^31.
- pnr_eval_image at the block-count switches, with subnormal / zero / negative / NaN depth_gt and NaN / Inf maps,
  each sum held to the bound of its own summation order; the Evaluator's frame buffer, workspace growth, reset() and
  a non-default stream.
"""
import functools
import math
import operator

import numpy as np
import pytest
import torch

from oracle import reference_eval as RE
from panopticnerf_b200 import _capi
from panopticnerf_b200.lib.evaluators import Evaluator, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TWO53 = 2 ** 53
IMAX, IMIN = 2 ** 31 - 1, -2 ** 31
IMAGE_BYTES = 8 * 256 * 6       # the image partials at the start of every workspace; the pair table follows


def dev(a, dtype=torch.int32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(dtype).to(DEV)


def run_semantic(pred, gt, C, table=None):
    conf = torch.zeros(C, C + 1, dtype=torch.int64, device=DEV)
    ops.eval_semantic(dev(pred).reshape(-1), dev(gt).reshape(-1), C, conf, None if table is None else dev(table))
    return conf.cpu().numpy().astype(np.uint64)


def new_tallies(C):
    return [torch.zeros(C, dtype=torch.int64, device=DEV) for _ in range(3)] + [
        torch.zeros(C, dtype=torch.float64, device=DEV)]


def run_panoptic(pred, gt, C, is_thing, table=None, acc=None, ws=None):
    """tp, fp, fn, iou_sum (device tensors, added to `acc` when given)."""
    acc = new_tallies(C) if acc is None else acc
    if ws is None:
        ws = torch.empty(ops.workspace_bytes(np.size(gt)), dtype=torch.uint8, device=DEV)
    ops.eval_panoptic(dev(pred).reshape(-1), dev(gt).reshape(-1), C, dev(is_thing, torch.uint8), ws, *acc,
                      None if table is None else dev(table))
    return acc


def host(acc):
    return [t.cpu().numpy() for t in acc]


def assert_tallies(got, ref):
    for name, a, b in zip(("tp", "fp", "fn", "iou_sum"), got, ref):
        assert np.array_equal(a, np.asarray(b)), (name, a, b)


def check_against_oracle(pred, gt, C, is_thing, table=None):
    """Semantic confusion and panoptic tallies of one frame, exact against the oracle; returns the oracle's tallies."""
    t64 = None if table is None else np.asarray(table, np.int64)
    assert np.array_equal(run_semantic(pred, gt, C, table), RE.semantic_confusion(pred, gt, C, t64))
    ref = RE.panoptic_frame(pred, gt, C, is_thing, t64)
    assert_tallies(host(run_panoptic(pred, gt, C, is_thing, table)), ref)
    return ref


# ------------------------------------------------------------------------------------------------ 128-bit IoU sum
# Dataset ids 0..299 -> channel 0 (300 000 panoptic ids), 300..304 -> channel 1, the rest of the table void.
IOU_C, IOU_THING = 2, [0, 0]
IOU_TABLE = np.full(400, -1, np.int32)
IOU_TABLE[:300] = 0
IOU_TABLE[300:305] = 1
CH1_SEGS = [(3, 4), (5, 7), (2, 3), (11, 13), (4, 4)]     # a few matches in channel 1, which must not mix with 0
# every IoU a / b with 2 <= b <= 64 and b / 2 < a <= b, and the multiple of 2^-53 it is as a double
CANDIDATES = [(a, b) for b in range(2, 65) for a in range(b // 2 + 1, b + 1)]


def q_of(a, b):
    return int(a / b * TWO53)          # a / b is correctly rounded, so this is the integer the kernel adds


def iou_frame(segs0, segs1=CH1_SEGS, seed=0):
    """(pred, gt): gt segment i has area b_i and is predicted as itself on a_i of its pixels and as void on the rest.
    The void pixels lie inside the gt, so they count towards its area and union = b_i: IoU = a_i / b_i exactly."""
    ab = list(segs0) + list(segs1)
    ids = np.concatenate([np.arange(len(segs0)), 300_000 + np.arange(len(segs1))])
    a = np.array([x for x, _ in ab], np.int64)
    b = np.array([y for _, y in ab], np.int64)
    gt = np.repeat(ids, b)
    pos = np.arange(gt.size) - np.repeat(np.cumsum(b) - b, b)
    pred = np.where(pos < np.repeat(a, b), gt, -1)
    perm = np.random.default_rng(seed).permutation(gt.size)
    return pred[perm].astype(np.int32), gt[perm].astype(np.int32)


def random_segs(count, seed):
    g = np.random.default_rng(seed)
    return [CANDIDATES[i] for i in g.integers(0, len(CANDIDATES), count)]


def ulp_exp(Q):
    """k such that 2^k is the spacing of doubles at the integer Q (Q >= 2^53)."""
    return Q.bit_length() - 53


@functools.lru_cache(maxsize=None)
def residue_layers(M):
    """The residues modulo M of sums of one and of two CANDIDATES' q, each with one way to reach it."""
    one = {}
    for i, (a, b) in enumerate(CANDIDATES):
        one.setdefault(q_of(a, b) % M, i)
    two = {}
    for r1, i in one.items():
        for r2, j in one.items():
            two.setdefault((r1 + r2) % M, (i, j))
    return one, two


def pick_residue(need, M):
    """Indices of one, two or three CANDIDATES whose q sum to `need` modulo M: a DP over residues, layers 1 and 2
    tabulated, layer 3 met in the middle."""
    one, two = residue_layers(M)
    if need in one:
        return [one[need]]
    if need in two:
        return list(two[need])
    for r1, i in one.items():
        if (need - r1) % M in two:
            return [i, *two[(need - r1) % M]]
    raise AssertionError(f"residue {need} mod {M} unreachable")


# The final rounding of the exact sum Q (in units of 2^-53), with 2^k the spacing of doubles at Q.  "above" has an
# even neighbour below and lies one unit above half: only the sticky bit of the 128-bit conversion rounds it up.
ROUNDINGS = {"tie_even": lambda k: 1 << (k - 1), "tie_odd": lambda k: (1 << k) | (1 << (k - 1)),
             "above": lambda k: (1 << (k - 1)) + 1, "below": lambda k: (1 << k) | ((1 << (k - 1)) - 1)}


@functools.lru_cache(maxsize=None)
def rounding_case(count, kind):
    """`count` channel-0 segments whose exact IoU sum falls on the rounding case `kind`."""
    for seed in range(20):
        segs = random_segs(count - 3, seed)
        Q0 = sum(q_of(a, b) for a, b in segs)
        k = ulp_exp(Q0 + 3 * TWO53)
        M = 1 << (k + 1)
        want = ROUNDINGS[kind](k)
        segs = segs + [CANDIDATES[i] for i in pick_residue((want - Q0) % M, M)]
        segs += [CANDIDATES[-1]] * (count - len(segs))                # IoU 1 (q = 2^53 = 0 mod M) fills up
        Q = sum(q_of(a, b) for a, b in segs)
        if ulp_exp(Q) == k:                                            # still in the binade the residue was picked for
            assert Q % M == want and len(segs) == count
            return tuple(segs)
    raise AssertionError("no seed kept the sum in one binade")


def count_case(count, kind):
    return tuple([CANDIDATES[-1]] * count) if kind == "one" else tuple(random_segs(count, count))


def sums_of(segs):
    """(exact integer sum Q, fsum, the left-to-right double sum, Q truncated to a double).  (Python's sum() of floats
    is compensated since 3.12, so the left-to-right sum is a reduce.)"""
    Q = sum(q_of(a, b) for a, b in segs)
    ious = [a / b for a, b in segs]
    k = max(ulp_exp(Q), 0)
    return Q, math.fsum(ious), functools.reduce(operator.add, ious, 0.0), ((Q >> k) << k) / TWO53


def check_iou_frame(segs0, seed=0):
    pred, gt = iou_frame(segs0, seed=seed)
    Q, fs, _, _ = sums_of(segs0)
    assert fs == Q / TWO53                                             # int / int is correctly rounded
    got = host(run_panoptic(pred, gt, IOU_C, IOU_THING, IOU_TABLE))
    want_tp = [len(segs0), len(CH1_SEGS)]
    assert_tallies(got, (want_tp, [0, 0], [0, 0], [fs, math.fsum(a / b for a, b in CH1_SEGS)]))
    return Q


@pytest.mark.parametrize("count,kind", [(2047, "one"), (2048, "one"), (2049, "one"), (4097, "one"), (2047, "mixed"),
                                        (4097, "mixed"), (2 ** 17 + 3, "mixed")])
def test_iou_sum_across_low_word_wraps(count, kind):
    """IoU 1 is q = 2^53: 2048 of them are exactly 2^64, the first wrap of the low word (to 0, with one carry)."""
    segs = count_case(count, kind)
    Q = check_iou_frame(segs, seed=count)
    if kind == "one":
        assert Q == count << 53
    if count >= 2 ** 17:
        assert Q >> 64 >= 16                                           # the high word spans >= 5 bits: shift > 1


@pytest.mark.parametrize("count", [1000, 3001, 2 ** 17 + 3])
@pytest.mark.parametrize("kind", sorted(ROUNDINGS))
def test_iou_sum_rounding_ties(count, kind):
    """~1000 matches round in the one-word branch, ~3000 in the two-word branch with a 1-bit shift, 2^17 + 3 with a
    6-bit shift (the unit one above half is then among the bits shifted out)."""
    segs = rounding_case(count, kind)
    Q = check_iou_frame(segs, seed=count + 1)
    assert (Q >> 64 == 0) == (count == 1000)


def test_iou_cases_discriminate():
    """Some case's fsum differs both from a left-to-right double sum and from the truncated 128-bit value: a kernel
    that sums IoUs with float atomics or truncates could not pass every case above."""
    cases = [rounding_case(c, k) for c in (1000, 3001, 2 ** 17 + 3) for k in ROUNDINGS]
    cases += [count_case(c, "mixed") for c in (2047, 4097, 2 ** 17 + 3)]
    both = 0
    for segs in cases:
        _, fs, naive, trunc = sums_of(segs)
        both += fs != naive and fs != trunc
    assert both >= 1
    for c in (1000, 3001, 2 ** 17 + 3):                               # rounding up: truncation is always wrong
        for k in ("tie_odd", "above"):
            _, fs, _, trunc = sums_of(rounding_case(c, k))
            assert fs != trunc


def test_iou_sum_of_two_frames():
    """Each frame is rounded once; the accumulator gets fl(fsum(frame 1) + fsum(frame 2))."""
    s1, s2 = rounding_case(3001, "tie_odd"), rounding_case(3001, "above")
    acc = new_tallies(IOU_C)
    for segs, seed in ((s1, 1), (s2, 2)):
        pred, gt = iou_frame(segs, seed=seed)
        run_panoptic(pred, gt, IOU_C, IOU_THING, IOU_TABLE, acc=acc)
    got = host(acc)
    ch1 = math.fsum(a / b for a, b in CH1_SEGS)
    assert_tallies(got, ([len(s1) + len(s2), 2 * len(CH1_SEGS)], [0, 0], [0, 0],
                         [sums_of(s1)[1] + sums_of(s2)[1], ch1 + ch1]))


# ------------------------------------------------------------------------------------------------ decision boundaries
# The closed-form frames of test_cpu_eval.py, as literal data: (pred, gt, is_thing, id table).  C = 4, channels 1 and
# 2 are things unless stated.
THING = [0, 1, 1, 0]
CLOSED_FORM = {
    "perfect": ([[0, 0, 1001, 1001, 1002], [3000, 3000, 2001, 2001, 2001]],
                [[0, 0, 1001, 1001, 1002], [3000, 3000, 2001, 2001, 2001]], THING, None),
    "split": ([1001] * 6 + [1002] * 4, [1001] * 10, THING, None),
    "iou_one_half": ([1001] * 5 + [1002] * 5, [1001] * 10, THING, None),
    "merged_two_fn": ([1003] * 10, [1001] * 5 + [1002] * 5, THING, None),
    "merged_one_match": ([1003] * 10, [1001] * 6 + [1002] * 4, THING, None),
    "void_in_union": ([1001] * 8, [1001] * 4 + [-1] * 4, THING, None),
    "void_more_than_half": ([0] * 10 + [3000] * 10, [0] * 10 + [-1] * 6 + [0] * 4, THING, None),
    "void_exactly_half": ([0] * 10 + [3000] * 10, [0] * 10 + [-1] * 5 + [0] * 5, THING, None),
    "unmapped_is_void": ([1001] * 8, [1001] * 4 + [9000] * 4, THING, None),
    "crowd_excuses": ([2001] * 10, [2000] * 6 + [0] * 4, THING, None),
    "crowd_of_another_class": ([1001] * 10, [2000] * 6 + [0] * 4, THING, None),
    "crowd_id_predicted": ([2000] * 6 + [0] * 4, [2000] * 6 + [0] * 4, THING, None),
    "crowd_on_itself": ([3000] * 10, [3000] * 10, [0, 1, 1, 1], None),
    "void_only": ([0, 1001, 2002, 3000, -1, 5, 7, 8, 9, 10], [-1] * 7 + [64000] * 3, THING, None),
    "no_table": ([0, 1001, 2000, -1, 9000, 0, 0], [0, 1001, 1002, 2000, 3000, -5, 7000], THING, None),
    "id_table": ([0, 1001, 2000, -1, 9000, 0, 0], [0, 1001, 1002, 2000, 3000, -5, 7000], THING, [2, -1, 0, 7]),
}


@pytest.mark.parametrize("name", sorted(CLOSED_FORM))
def test_closed_form_frames(name):
    pred, gt, thing, table = CLOSED_FORM[name]
    check_against_oracle(np.array(pred), np.array(gt), 4, thing, table)


def match_frame(inter, uni, void):
    """gt 1001 (area g) predicted as 1002 on `inter` of its pixels and as void on the rest; 1002 also covers e pixels
    of stuff gt 0 and `void` pixels of void gt: union = (inter + e + void) + g - inter - void = g + e = uni."""
    e = (uni - inter) // 2
    g = uni - e
    gt = [1001] * g + [0] * e + [-1] * void
    pred = [1002] * inter + [-1] * (g - inter) + [1002] * (e + void)
    return np.array(pred), np.array(gt)


@pytest.mark.parametrize("inter", [1, 2, 3, 50, 999, 2 ** 15, 2 ** 16 + 1])
@pytest.mark.parametrize("void", [False, True])
def test_match_boundary(inter, void):
    """2 inter == union is not a match; 2 inter == union + 1 is.  With void pixels under the prediction, the union
    only comes out right when |p ∩ void| is taken out of it."""
    for uni, match in ((2 * inter, False), (2 * inter - 1, True)):
        if uni < inter:
            continue
        pred, gt = match_frame(inter, uni, inter // 2 + 1 if void else 0)
        tp = check_against_oracle(pred, gt, 4, THING)[0]
        assert tp[1] == int(match), (uni, tp)


@pytest.mark.parametrize("s,kind", [(s, k) for k in ("void", "crowd", "both") for s in (1, 2, 3, 64, 1001, 2 ** 16 + 1)
                                    if (s, k) != (1, "both")])
def test_false_positive_excuse_boundary(s, kind):
    """Prediction 2005 (thing channel 2) lies on `void` void pixels, `crowd` pixels of the crowd 2000 of its class and
    `rest` pixels of stuff 0.  2 ignored == area is a false positive; 2 ignored == area + 1 is excused.  "both": void
    and crowd each stay at most half of the area, only their sum crosses it."""
    void = {"void": s, "crowd": 0, "both": (s + 1) // 2}[kind]
    crowd = s - void
    for rest, fp in ((s, 1), (s - 1, 0)):
        gt = np.array([-1] * void + [2000] * crowd + [0] * rest)
        pred = np.full(gt.size, 2005)
        got = check_against_oracle(pred, gt, 4, THING)
        assert got[1][2] == fp and got[0].sum() == 0, (rest, got)
        if kind == "both":
            assert 2 * void <= gt.size and 2 * crowd <= gt.size


# ------------------------------------------------------------------------------------------------ hash tables
M1, M2, S33 = np.uint64(0xff51afd7ed558ccd), np.uint64(0xc4ceb9fe1a85ec53), np.uint64(33)


def mix64(k):
    """The kernels' murmur3 finaliser on uint64 keys, truncated to uint32 (eval_kernels.cu mix64)."""
    k = k ^ (k >> S33)
    k = k * M1
    k = k ^ (k >> S33)
    k = k * M2
    k = k ^ (k >> S33)
    return k & np.uint64(0xFFFFFFFF)


def seg_key(ids):
    return np.asarray(ids, np.int64).astype(np.uint32).astype(np.uint64)


def pair_key(g, p):
    return (seg_key(g) << np.uint64(32)) | seg_key(p)


def table_slots(n):
    S = 1024
    while S < 2 * n:
        S *= 2
    return S


def tables_of(ws, S):
    """The pair, gt and pred key tables of a workspace after a call (layout of eval_kernels.cu carve())."""
    w = ws[IMAGE_BYTES:IMAGE_BYTES + 16 * S]
    pair = w[:8 * S].view(torch.int64).cpu().numpy().view(np.uint64)
    gtk = w[8 * S:12 * S].view(torch.int32).cpu().numpy().view(np.uint32).astype(np.uint64)
    prk = w[12 * S:].view(torch.int32).cpu().numpy().view(np.uint32).astype(np.uint64)
    return pair, gtk, prk


EMPTY64, EMPTY32 = np.uint64(2 ** 64 - 1), np.uint64(2 ** 32 - 1)


@pytest.mark.parametrize("n", [512, 513, 2 ** 16, 2 ** 20])
def test_tables_at_their_fullest(n):
    """n pixels, each its own gt and pred segment: n distinct pairs, gt ids and pred ids, so at n = 512, 2^16, 2^20
    (S = 2n) all three tables are exactly half full, and at 513 the first past a doubling (S = 2048).  Dataset ids up
    to 2137 go through a table d -> d % 64.  Half the pixels predict their gt id (IoU 1: a match), the others the id
    + 1 089 000, which is the next channel (an FN and an FP)."""
    C, O = 64, 1089 * 1000
    table = (np.arange(2200) % C).astype(np.int32)
    g = np.random.default_rng(n)
    gt = g.permutation(n)
    same = g.random(n) < 0.5
    pred = np.where(same, gt, gt + O)
    S = table_slots(n)
    assert S == (2048 if n == 513 else 2 * n)
    ws = torch.empty(ops.workspace_bytes(n), dtype=torch.uint8, device=DEV)
    got = host(run_panoptic(pred, gt, C, np.zeros(C), table, ws=ws))
    cg, cp = table[gt // 1000], table[pred // 1000]
    assert not (cg[~same] == cp[~same]).any()
    tp = np.bincount(cg[same], minlength=C)
    assert_tallies(got, (tp, np.bincount(cp[~same], minlength=C), np.bincount(cg[~same], minlength=C), tp.astype(float)))
    pair, gtk, prk = tables_of(ws, S)
    assert [(pair != EMPTY64).sum(), (gtk != EMPTY32).sum(), (prk != EMPTY32).sum()] == [n, n, n]
    if n <= 2 ** 16:
        ref = RE.panoptic_frame(pred, gt, C, np.zeros(C), table.astype(np.int64))
        assert_tallies(got, ref)


WRAP_C, WRAP_THING = 3, [0, 1, 0]
WRAP_TABLE = (np.arange(2 ** 17) % WRAP_C).astype(np.int32)          # ids below 1.31e8 have a channel


def ids_homing_last8(S, count, start):
    """The first `count` ids >= start whose segment key's home slot (mix64(key) & (S - 1)) is in [S - 8, S)."""
    out, lo, step = [], start, 1 << 22
    while len(out) < count:
        ids = np.arange(lo, lo + step, dtype=np.int64)
        out.extend(ids[mix64(seg_key(ids)) & np.uint64(S - 1) >= np.uint64(S - 8)].tolist())
        lo += step
    return np.array(out[:count], np.int64)


def pairs_homing_last8(S, gts):
    """Every (gt id, pred id) with the gt id from `gts` and the pred id in [0, S / 8) whose pair key's home slot is in
    [S - 8, S): about one per gt id."""
    g_out, p_out = [], []
    p = np.arange(S // 8, dtype=np.int64)
    for g in gts.tolist():
        hit = p[mix64(pair_key(np.full(p.size, g), p)) & np.uint64(S - 1) >= np.uint64(S - 8)]
        g_out += [g] * hit.size
        p_out += hit.tolist()
    return np.array(g_out, np.int64), np.array(p_out, np.int64)


@pytest.mark.parametrize("n,K", [(512, 120), (2 ** 16, 200), (2 ** 20, 200)])
def test_probe_chains_wrap_around(n, K):
    """Keys picked on the host so that every one of them hashes to one of the last 8 slots [S - 8, S) of its table
    (S = 1024, 2^17, 2^21): K gt ids (gt table), K pred ids (pred table) and ~K (gt, pred) pairs (pair table).
    Each table then holds a probe chain of ~K slots that starts in its last 8 slots and wraps to slot 0.  The rest of
    the frame is void on both sides (never inserted)."""
    S = table_slots(n)
    G = ids_homing_last8(S, K, 0)
    P = ids_homing_last8(S, K, 50_000_000)
    Gq, Pq = pairs_homing_last8(S, G)
    assert Gq.size >= K // 2
    # every pair (Gq, Pq) twice, then (G[i], P[i]) once: pred P[i] overlaps gt G[i] -> some same-channel matches
    gt = np.concatenate([Gq, Gq, G])
    pred = np.concatenate([Pq, Pq, P])
    assert gt.size <= n
    perm = np.random.default_rng(n).permutation(n)
    gt = np.concatenate([gt, np.full(n - gt.size, -1)])[perm]
    pred = np.concatenate([pred, np.full(n - pred.size, -1)])[perm]
    ws = torch.empty(ops.workspace_bytes(n), dtype=torch.uint8, device=DEV)
    got = host(run_panoptic(pred, gt, WRAP_C, WRAP_THING, WRAP_TABLE, ws=ws))
    assert_tallies(got, RE.panoptic_frame(pred, gt, WRAP_C, WRAP_THING, WRAP_TABLE.astype(np.int64)))
    assert got[0].sum() > 0 and got[1].sum() > 0 and got[2].sum() > 0
    # The device put the keys where the mirror of mix64 says: at most 8 of them fit in [S - 8, S), and every other one
    # sits past the wrap, in a slot below the table's count of occupied slots (its probe ran from its home through
    # S - 1 and 0 over occupied slots only).  A wrong mirror would scatter them over the whole table.
    for table, keys, empty in zip(tables_of(ws, S), (pair_key(Gq, Pq), seg_key(G), seg_key(P)),
                                  (EMPTY64, EMPTY32, EMPTY32)):
        assert (mix64(keys) & np.uint64(S - 1) >= np.uint64(S - 8)).all()
        occupied = np.flatnonzero(table != empty)
        slot = dict(zip(table[occupied].tolist(), occupied.tolist()))
        where = np.array([slot[k] for k in keys.tolist()])
        wrapped = where < S - 8
        assert wrapped.sum() >= keys.size - 8 and where[wrapped].max() < occupied.size


# ------------------------------------------------------------------------------------------------ id edges
ID_C = 64
EDGE_IDS = [IMAX, IMIN, -1, -1000, 0, 7, 1005, 2005, 3005, 63 * 1000 + 9, 63 * 1000, 64 * 1000 + 9, 99 * 1000 + 5,
            100 * 1000 + 5, 2147483 * 1000, 12 * 1000 + 1]


def edge_table(kind):
    """None: channel d for d < 64.  "short": 100 entries, d % 64, with entry 1 = -1, 2 = C - 1, 3 = C.  "long": the
    same first 100 entries, then -1 up to the 2 147 484th entry, which maps INT32_MAX (and 2147483000) to channel 7."""
    if kind is None:
        return None
    t = np.full(100 if kind == "short" else IMAX // 1000 + 1, -1, np.int32)
    t[:100] = np.arange(100) % ID_C
    t[1], t[2], t[3] = -1, ID_C - 1, ID_C
    if kind == "long":
        t[-1] = 7
    return t


@pytest.mark.parametrize("thing", ["all", "none"])
@pytest.mark.parametrize("table", [None, "short", "long"])
def test_id_edges(table, thing):
    """Every (gt, pred) combination of the edge ids, 1 .. 4 pixels each, plus 200 pixels of (e, e) for every other
    edge id so that its segments match."""
    E = np.array(EDGE_IDS, np.int64)
    i, j = np.meshgrid(np.arange(E.size), np.arange(E.size), indexing="ij")
    cnt = 1 + (i * 7 + j * 3) % 4 + np.where((i == j) & (i % 2 == 0), 200, 0)
    gt = np.repeat(E[i.ravel()], cnt.ravel())
    pred = np.repeat(E[j.ravel()], cnt.ravel())
    perm = np.random.default_rng(1).permutation(gt.size)
    gt, pred = gt[perm].astype(np.int32), pred[perm].astype(np.int32)
    is_thing = np.full(ID_C, thing == "all")
    t = edge_table(table)
    ref = check_against_oracle(pred, gt, ID_C, is_thing, t)
    assert ref[0].sum() > 0 and ref[2].sum() > 0
    if table == "long":
        ch = RE.channels(np.array([IMAX, 2147483000]), ID_C, t.astype(np.int64))
        assert ch.tolist() == [7, 7]


# ------------------------------------------------------------------------------------------------ large frames
def test_panoptic_frame_of_2_24_pixels():
    """4096 x 4096: gt 1001 everywhere but a blocky band of 16 x 16 blocks (rows 0..255) and a void patch; the
    prediction shifts the band, relabels 10 % of its blocks, predicts void over a 256 x 1024 part of 1001 and 1001 over
    the void patch.  The (1001, 1001) pair alone counts ~15.6 M pixels."""
    H = W = 4096
    C = 64
    is_thing = np.arange(C) % 2 == 1
    g = np.random.default_rng(24)
    band_ids = g.integers(0, C, (16, 256)) * 1000 + g.integers(0, 1000, (16, 256))
    gt = np.full((H, W), 1001, np.int64)
    gt[:256] = np.repeat(np.repeat(band_ids, 16, 0), 16, 1)
    gt[512:768, :512] = -1
    relabel = np.where(g.random(band_ids.shape) < 0.1, g.integers(0, C, band_ids.shape) * 1000 + 3, band_ids)
    pred = np.full((H, W), 1001, np.int64)
    pred[:256] = np.roll(np.repeat(np.repeat(relabel, 16, 0), 16, 1), (2, 1), (0, 1))
    pred[256:512, :1024] = -1
    gt, pred = gt.astype(np.int32), pred.astype(np.int32)
    torch.cuda.reset_peak_memory_stats()
    ref = check_against_oracle(pred, gt, C, is_thing)
    print(f"n = 2^24: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB "
          f"(workspace {ops.workspace_bytes(H * W) / 2 ** 30:.2f} GiB)")
    assert ref[0][1] >= 1 and ref[0].sum() > 100 and ref[1].sum() > 0 and ref[2].sum() > 0


def test_semantic_frame_of_2_31_minus_1_pixels():
    """n = 2^31 - 1, the largest accepted: gt = buf[0:n], pred = buf[1:n + 1] of one int32 buffer of 2^31 pixels,
    filled on the device with a tile of L = 1000 ids in runs of two (dataset ids -1 .. 64, so void gt, void
    predictions, every channel, diagonal and off-diagonal bins).  Pixel i pairs tile[i % L] with tile[(i + 1) % L]:
    each tile position j occurs floor(n / L) times, plus once for j < n % L, and the confusion matrix is the sum of
    those counts."""
    n, L, C = 2 ** 31 - 1, 1000, 64
    need = (n + 1) * 4
    free, _ = torch.cuda.mem_get_info()
    if free < need + 2 ** 30:
        pytest.skip(f"an int32 buffer of 2^31 pixels needs {need / 2 ** 30:.1f} GiB; {free / 2 ** 30:.1f} GiB free "
                    "on this device (shared)")
    j = np.arange(L)
    tile = ((j // 2 % (C + 2) - 1) * 1000 + j % 13).astype(np.int32)
    torch.cuda.reset_peak_memory_stats()
    buf = torch.empty(n + 1, dtype=torch.int32, device=DEV)
    k, r = divmod(n + 1, L)
    t = dev(tile)
    buf[:k * L].view(k, L).copy_(t.expand(k, L))
    buf[k * L:] = t[:r]
    conf = torch.zeros(C, C + 1, dtype=torch.int64, device=DEV)
    ops.eval_semantic(buf[1:], buf[:n], C, conf)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    del buf, t
    torch.cuda.empty_cache()
    q, rem = divmod(n, L)
    count = q + (j < rem)
    gch = RE.channels(tile, C)
    pch = RE.channels(np.roll(tile, -1), C)
    want = np.zeros((C, C + 1), np.uint64)
    keep = gch >= 0
    np.add.at(want, (gch[keep], np.where(pch < 0, C, pch)[keep]), count[keep].astype(np.uint64))
    print(f"n = 2^31 - 1: peak device memory {peak / 2 ** 30:.2f} GiB")
    assert np.array_equal(conf.cpu().numpy().astype(np.uint64), want)
    assert want[:, C].sum() > 0 and np.trace(want[:, :C]) > 0 and want.sum() > 2 ** 31 * 0.9


def test_first_refused_size_launches_nothing():
    """n = 2^31 is refused with PNR_ERR_ARG before any launch, so the accumulators stay untouched."""
    lib = _capi.lib()
    x = torch.zeros(16, dtype=torch.int32, device=DEV)
    conf = torch.zeros(4, 5, dtype=torch.int64, device=DEV)
    tal = new_tallies(4)
    ws = torch.empty(ops.workspace_bytes(16), dtype=torch.uint8, device=DEV)
    rc = lib.pnr_eval_semantic(x.data_ptr(), x.data_ptr(), 2 ** 31, 4, None, 0, conf.data_ptr(), None)
    assert rc == -1 and b"n=2147483648" in lib.pnr_last_error()
    th = dev([0, 1, 0, 0], torch.uint8)
    rc = lib.pnr_eval_panoptic(x.data_ptr(), x.data_ptr(), 2 ** 31, 4, None, 0, th.data_ptr(), ws.data_ptr(),
                               ws.numel(), *[a.data_ptr() for a in tal], None)
    assert rc == -1 and b"n=2147483648" in lib.pnr_last_error()
    torch.cuda.synchronize()
    assert int(conf.abs().sum()) == 0 and all(float(a.abs().sum()) == 0 for a in tal)


# ------------------------------------------------------------------------------------------------ image / depth
U = 2.0 ** -53


def image_terms(rgb, rgb_gt, depth, depth_gt):
    """The float64 terms the kernel adds: (rgb - gt)^2 per channel; |d|, d^2, |d| / gt over gt > 0."""
    d = rgb.astype(np.float64) - rgb_gt.astype(np.float64)
    g = depth_gt.astype(np.float64)
    ok = g > 0
    dd = depth.astype(np.float64)[ok] - g[ok]
    return [d * d, np.abs(dd), dd * dd, np.abs(dd) / g[ok]]


def summation_bound(n):
    """Roundings on the path of one term through pnr_eval_image: its thread's sequential sum (`per` terms: 3 per
    pixel for rgb), the block's 8-level tree, the finish kernel's 8-level tree, and the product (which the kernel may
    fuse into its add) - so |got - exact| <= (per_thread + 17) 2^-53 sum |t| for the non-negative terms, with one
    spare rounding for the reference's own extended-precision sum."""
    blocks = min(-(-n // 256), 256)
    per_thread = -(-n // (blocks * 256))
    return [(3 * per_thread + 17) * U, (per_thread + 17) * U, (per_thread + 17) * U, (per_thread + 17) * U]


def check_image(n, rgb, rgb_gt, depth, depth_gt):
    ws = torch.empty(ops.workspace_bytes(0), dtype=torch.uint8, device=DEV)
    s = torch.zeros(6, dtype=torch.float64, device=DEV)
    ops.eval_image(s, ws, dev(rgb, torch.float32), dev(rgb_gt, torch.float32), dev(depth, torch.float32),
                   dev(depth_gt, torch.float32))
    got = s.cpu().numpy()
    ref = RE.image_sums(rgb, rgb_gt, depth, depth_gt)
    assert got[1] == n and got[5] == ref[5] == int((depth_gt.astype(np.float64) > 0).sum())
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(np.isinf(got), np.isinf(ref))
    if np.isfinite(ref).all():
        assert np.finfo(np.longdouble).nmant >= 63
        worst = 0.0
        for k, t, rel in zip((0, 2, 3, 4), image_terms(rgb, rgb_gt, depth, depth_gt), summation_bound(n)):
            exact = np.sum(t.astype(np.longdouble))
            err = abs(np.longdouble(got[k]) - exact)
            bound = rel * np.sum(np.abs(t).astype(np.longdouble))
            assert err <= bound, (k, float(err), float(bound))
            worst = max(worst, float(err / bound) if bound > 0 else 0.0)
        print(f"n = {n}: largest error / bound = {worst:.3e}")
    return got, ref


def image_frame(n, seed):
    g = np.random.default_rng(seed)
    rgb, rgb_gt = g.random((n, 3), np.float32), g.random((n, 3), np.float32)
    depth = (g.random(n, np.float32) * 80).astype(np.float32)
    depth_gt = np.where(g.random(n) < 0.3, 0, g.random(n, np.float32) * 80).astype(np.float32)
    depth_gt = np.where(g.random(n) < 0.05, -1, depth_gt).astype(np.float32)
    return rgb, rgb_gt, depth, depth_gt


@pytest.mark.parametrize("n", [1, 255, 256, 257, 65535, 65536, 65537, 2 ** 24 + 3])
def test_image_sums_within_their_summation_bound(n):
    """n <= 65536 has one pixel per thread; 65537 the first thread with two; 2^24 + 3 has 257 per thread."""
    check_image(n, *image_frame(n, n))


def test_image_depth_gt_edges():
    """depth_gt of 1e-38 (an fp32 subnormal), 1e-45 (the smallest, 2^-149), 0, negative and NaN: the subnormals are
    positive and counted, the rest skipped (NaN > 0 is false)."""
    rgb, rgb_gt, depth, depth_gt = image_frame(300, 7)
    depth_gt[:6] = np.array([1e-38, 1e-45, 0.0, -0.0, -2.5, np.nan], np.float32)
    depth[:6] = 5.0
    assert depth_gt[1] > 0
    got, ref = check_image(300, rgb, rgb_gt, depth, depth_gt)
    assert got[5] == int((depth_gt[6:] > 0).sum()) + 2


@pytest.mark.parametrize("where,value", [("rgb", np.nan), ("rgb", np.inf), ("depth", np.nan), ("depth", -np.inf),
                                         ("rgb_gt", -np.inf), ("depth_gt", np.inf)])
def test_image_non_finite_maps(where, value):
    """A NaN or Inf in a map makes its sums NaN or Inf as numpy's are; the other sums and the counts are unchanged.
    An infinite depth_gt is positive, so it is counted: d = -inf, |d| / gt = inf / inf = NaN."""
    maps = dict(zip(("rgb", "rgb_gt", "depth", "depth_gt"), image_frame(1000, 3)))
    maps["depth_gt"][:20] = 7.0
    m = maps[where]
    m.reshape(-1)[11] = value
    got, ref = check_image(1000, maps["rgb"], maps["rgb_gt"], maps["depth"], maps["depth_gt"])
    assert not np.isfinite(ref).all()


def test_perfect_frame_psnr_is_infinite():
    n, C = 777, 3
    g = np.random.default_rng(0)
    rgb = dev(g.random((n, 3), np.float32), torch.float32)
    ids = dev(g.integers(0, C, n) * 1000)
    ev = Evaluator(num_classes=C)
    ev.evaluate({"rgb_map": rgb}, {"panoptic_gt": ids, "panoptic_pred": ids, "rgb": rgb.clone()})
    got = ev.summarize()
    assert got["psnr"] == math.inf and got["pq"] == 1.0 and got["miou"] == 1.0
    fs = ev.frame_sums[:1].cpu().numpy()
    assert RE.summarize(ev.conf.cpu().numpy(), *host((ev.tp, ev.fp, ev.fn, ev.iou_sum)), np.zeros(C), fs)["psnr"] == math.inf


# ------------------------------------------------------------------------------------------------ Evaluator
EV_C = 19
EV_THING = np.arange(EV_C) % 3 == 1
EV_SIZES = [(24, 40), (48, 64), (72, 96)]
EV_ORDER = [0] * 26 + [1] * 26 + [2] * 26 + [1] * 26 + [0] * 26          # 130 frames: growing, then shrinking


def blocky_frame(H, W, seed):
    """8 x 8 blocks of ids of the 19 channels (crowd, void and unmapped blocks among them); the prediction is the gt
    shifted by one pixel with 15 % of its blocks relabelled."""
    g = np.random.default_rng(seed)
    nby, nbx = -(-H // 8), -(-W // 8)
    d = g.integers(0, EV_C + 1, (nby, nbx))
    ids = d * 1000 + np.where(g.random(d.shape) < 0.1, 0, g.integers(1, 1000, d.shape))
    ids = np.where(g.random(d.shape) < 0.05, -1, ids)
    gt = np.repeat(np.repeat(ids, 8, 0), 8, 1)[:H, :W]
    relabel = np.where(g.random(d.shape) < 0.15, g.integers(0, EV_C, d.shape) * 1000 + 5, ids)
    pred = np.roll(np.repeat(np.repeat(relabel, 8, 0), 8, 1)[:H, :W], (1, 1), (0, 1))
    n = H * W
    rgb, rgb_gt = g.random((n, 3), np.float32), g.random((n, 3), np.float32)
    depth, depth_gt = (g.random(n, np.float32) * 50).astype(np.float32), (g.random(n, np.float32) * 60 - 10).astype(np.float32)
    return pred.astype(np.int32), gt.astype(np.int32), rgb, rgb_gt, depth, depth_gt


@functools.lru_cache(maxsize=None)
def ev_pool():
    """4 frames of each size, and the oracle's tallies and image sums of each."""
    pool = []
    for s, (H, W) in enumerate(EV_SIZES):
        for k in range(4):
            f = blocky_frame(H, W, 10 * s + k)
            pool.append((f, RE.semantic_confusion(f[0], f[1], EV_C), RE.panoptic_frame(f[0], f[1], EV_C, EV_THING),
                         RE.image_sums(*f[2:])))
    return pool


def ev_frames(lo=0, hi=len(EV_ORDER)):
    return [4 * EV_ORDER[i] + i % 4 for i in range(lo, hi)]


def run_evaluator(frames, stream=None, reset_after=None):
    pool = ev_pool()
    dev_frames = {}
    ev = Evaluator(num_classes=EV_C, is_thing=EV_THING)
    for i in set(frames):
        pred, gt, rgb, rgb_gt, depth, depth_gt = pool[i][0]
        dev_frames[i] = ({"rgb_map": dev(rgb, torch.float32), "depth_map": dev(depth, torch.float32)},
                         {"panoptic_gt": dev(gt), "panoptic_pred": dev(pred), "rgb": dev(rgb_gt, torch.float32),
                          "depth": dev(depth_gt, torch.float32)})
    if stream is not None:
        stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for k, i in enumerate(frames):
            if k == reset_after:
                ev.reset()
            ev.evaluate(*dev_frames[i])
    torch.cuda.synchronize()
    return ev


def accumulators(ev):
    return [t.cpu().clone() for t in (ev.conf, ev.tp, ev.fp, ev.fn, ev.iou_sum, ev.frame_sums[:ev.frames])]


def test_evaluator_bookkeeping():
    """130 frames of three sizes, growing then shrinking (the workspace is reallocated twice, the frame buffer
    doubles at 64 and 128), on a non-default stream: counts exact, iou_sum bit-equal to adding each frame's fsum in
    order, frame sums and metrics vs the oracle.  Bit-identical to the same frames on the default stream.  reset()
    after frame 70 leaves exactly what frames 70..129 give a fresh Evaluator."""
    pool, frames = ev_pool(), ev_frames()
    side = torch.cuda.Stream()
    ev = run_evaluator(frames, stream=side)
    assert ev.frames == 130 and ev.frame_sums.shape[0] == 256 and float(ev.frame_sums[130:].abs().sum()) == 0.0
    assert ev._ws.numel() == ops.workspace_bytes(72 * 96)
    conf = sum(pool[i][1] for i in frames)
    tp, fp, fn = (sum(pool[i][2][k] for i in frames) for k in range(3))
    iou = np.zeros(EV_C)
    for i in frames:
        iou = iou + pool[i][2][3]                                       # += per frame, in frame order
    sums = np.stack([pool[i][3] for i in frames])
    got = accumulators(ev)
    assert np.array_equal(got[0].numpy().astype(np.uint64), conf)
    assert_tallies([t.numpy() for t in got[1:5]], (tp, fp, fn, iou))
    np.testing.assert_allclose(got[5].numpy(), sums, rtol=1e-12, atol=0)
    ref = RE.summarize(conf, tp, fp, fn, iou, EV_THING, sums)
    res = ev.summarize()
    assert set(res) == set(ref) and res["frames"] == 130
    for k in ref:
        np.testing.assert_allclose(np.asarray(res[k], np.float64), np.asarray(ref[k], np.float64), rtol=1e-12, err_msg=k)
    assert tp.sum() > 0 and fp.sum() > 0 and fn.sum() > 0
    default = accumulators(run_evaluator(frames))
    assert all(torch.equal(a, b) for a, b in zip(got, default))
    after_reset = run_evaluator(frames, reset_after=70)
    assert after_reset.frames == 60
    fresh = accumulators(run_evaluator(frames[70:]))
    assert all(torch.equal(a, b) for a, b in zip(accumulators(after_reset), fresh))
