"""CPU tests of the fused MoE decode kernel's schedule model (tests/fused_schedule.py) and of the per-tile metric that
tests/test_gpu_moe_fused_branches.py applies to the kernel.

  * Random shapes and routings at G = 132 and 114 SMs: every (tile, k-iteration) is covered exactly once, a CTA starts at
    most one split part at k = 0 and at most one at k != 0 per segment (the partials slot rule), the first contributor
    owns k = 0, and the chunk table fits whenever fused_supported holds.
  * Every case of the GPU matrix reaches the branches it names at G = 132 (an H100 SXM).
  * Faults of the stream-K schedule injected into the float64 mirror (tests/fused_oracle.py) at the weakest point of each
    case score at least 4x the case's threshold: the metric would see them in the kernel.
"""
from __future__ import annotations

import random

import pytest

import fused_oracle as FO
import fused_schedule as FS
from test_gpu_moe_fused_branches import CASES, H100_SMS, THRESH, case_inputs, case_routing

MARGIN = 4.0


# ------------------------------------------------------------------------------------------ the model itself
def _random_launch(rng: random.Random):
    fmt = rng.choice(FS.FORMATS)
    w4 = fmt in FS.W4
    gated = True if w4 else rng.random() < 0.6
    H = 128 * rng.choice([2, 4, 8, 9, 16, 32, 56] if not w4 else [2, 4, 8, 16, 32, 56])
    I = 128 * rng.choice([1, 2, 3, 4, 12, 16, 32])
    E = rng.choice([1, 2, 4, 8, 16, 64, 128, 256, 512])
    M = rng.choice([1, 2, 3, 4, 5, 8, 16, 17, 31, 32, 33, 48, 64, 100, 256])
    k = rng.choice([1, 2, 4, 6, 8])
    skip = rng.choice([0.0, 0.0, 0.3, 0.9])
    hot = rng.random() < 0.3                     # a few experts take most slots: chunks of many rows
    pool = list(range(min(E, 4) if hot else E))
    ids = []
    for _ in range(M):
        row = rng.sample(pool + [-1] * k, k) if len(pool) >= k else [rng.choice(pool) for _ in range(k)]
        ids.append([e if rng.random() >= skip else -1 for e in row])
    return FS.Geometry(fmt, E, H, I, gated), ids


@pytest.mark.parametrize("G", [132, 114])
def test_schedule_invariants_random(G):
    rng = random.Random(1234 + G)
    n_fused = 0
    labels = set()
    for _ in range(500):
        geo, ids = _random_launch(rng)
        for align in (60, 0):
            sch = FS.build(geo, ids, G, align)
            FS.check_invariants(sch)
            labels |= sch.labels
            n_fused += sch.supported
    assert n_fused > 400
    # the sweep itself reaches the stream-K branches it is meant to check
    for lab in ("g1_split", "g2_split", "g1_aligned", "g2_aligned", "g2_unpaired", "g1_half_iter", "g2_half_iter",
                "g1_fix_small_multi", "ng1", "ng2", "no_rows", "grouped_gemm"):
        assert lab in labels, lab


def test_part_owner_is_the_inverse_of_part_start():
    for n in (1, 7, 56, 131, 132, 133, 1000, 7392):
        for parts in (1, 3, 114, 132):
            if parts > n:
                continue
            for c in range(parts):
                for i in range(FS.part_start(c, n, parts), FS.part_start(c + 1, n, parts)):
                    assert FS.part_owner(i, n, parts) == c


def test_fused_supported_bounds_the_chunk_table():
    """fused_supported's chunk bound (act + slots / 16) holds for the worst routing of every accepted shape."""
    for E in (1, 8, 64, 256, 512):
        for M in (1, 16, 17, 32, 33, 64, 128, 256):
            for k in (1, 2, 8):
                geo = FS.Geometry("bf16", E, 512, 256)
                if not FS.fused_supported(geo, M, k):
                    continue
                tn = FS.tn_max(geo, M)
                # most chunks: every active expert gets rows just past a chunk boundary
                n_act = min(E, M * k)
                ids = [[(t * k + j) % n_act for j in range(k)] for t in range(M)]
                chunks, _ = FS.chunk_table(geo, ids, tn)
                assert len(chunks) <= FS.FUSED_MAX_CHUNKS


def test_odd_hidden_tiles_never_fuse_for_4bit():
    for fmt in FS.W4:
        assert not FS.fused_supported(FS.Geometry(fmt, 8, 1152, 256), 4, 2)
    assert FS.fused_supported(FS.Geometry("bf16", 8, 1152, 256), 4, 2)


# ------------------------------------------------------------------------------------------ the GPU matrix
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_case_reaches_its_branches(name):
    c = CASES[name]
    _, ids, _ = case_routing(c)
    sch = FS.build(FS.Geometry(c.fmt, c.E, c.H, c.I, c.gated), ids, H100_SMS, c.align_g1)
    FS.check_invariants(sch)
    assert "fused" in sch.labels
    missing = set(c.labels) - sch.labels
    assert not missing, f"{name} does not reach {sorted(missing)} at G = {H100_SMS}"


# ------------------------------------------------------------------------------------------ fault injection
def _fault_candidates(m: FO.Mirror, sch: FS.Schedule, limit: int = 24):
    """{fault kind: [Fault]} at every place of the case where that fault can happen (at most `limit` per kind, spread
    over the launch).  Where a fault has a choice of k-block, the one whose partial product is smallest is taken."""
    geo = sch.geo
    out = {}

    def spread(lst):
        if len(lst) <= limit:
            return lst
        step = len(lst) / limit
        return [lst[int(i * step)] for i in range(limit)]

    g1 = [t for t in sch.tiles if t.ph == 0]
    drop1 = []
    for t in spread(g1):
        cols = FO._tile_cols(sch, 0, t.j)
        P = m._p1_of(t.q)[:, :, cols]
        norms = P.flatten(1).norm(dim=1)
        # one k-iteration of this tile lost: the k-blocks it loads
        ki = min(range(t.KI), key=lambda i: float(sum(norms[kb] for kb in sch.kblocks(0, i, i + 1))))
        drop1.append(FO.Fault(0, t.q, t.j, "drop", tuple(sch.kblocks(0, ki, ki + 1))))
    out["g1_kblock_dropped"] = drop1
    split2 = [t for t in sch.tiles if t.ph == 1 and t.split]
    if split2:
        out["g2_contributor_dropped"] = [
            FO.Fault(1, t.q, t.j, "drop", tuple(sch.kblocks(1, *min(((k0, k1) for _, k0, k1 in t.parts),
                                                                    key=lambda r: r[1] - r[0]))))
            for t in spread(split2)]
    split = [t for t in sch.tiles if t.split]
    if split:
        out["contributor_counted_twice"] = [
            FO.Fault(t.ph, t.q, t.j, "double", tuple(sch.kblocks(t.ph, *min(((k0, k1) for _, k0, k1 in t.parts),
                                                                         key=lambda r: r[1] - r[0]))))
            for t in spread(split)]
    if not sch.pair2:
        out["g2_neighbour_columns"] = [FO.Fault(1, t.q, t.j, "neighbour") for t in spread(
            [t for t in sch.tiles if t.ph == 1 and t.j + 1 < geo.J2])]
    half = [t for t in sch.tiles if t.half]
    if half:
        out["half_iteration_offset"] = []
        for t in spread(half):
            KB = geo.KB1 if t.ph == 0 else geo.KB2
            out["half_iteration_offset"].append(FO.Fault(t.ph, t.q, t.j, "shift", (KB - 1, KB - 2)))
    return out


FAULT_CASES = [n for n, c in CASES.items() if c.routing[0] != "none"]


@pytest.mark.parametrize("name", FAULT_CASES)
def test_injected_faults_exceed_threshold(name):
    c = CASES[name]
    layer, hidden, ids, w = case_inputs(c)
    sch = FS.build(layer.geo, ids, H100_SMS, c.align_g1)
    m = FO.Mirror(layer, sch, hidden, w)
    clean = m.out()
    thr = THRESH[(c.fmt, "f32")]
    cands = _fault_candidates(m, sch)
    assert cands
    report = {}
    for kind, faults in cands.items():
        assert faults, kind
        report[kind] = min(FO.max_tile_error(m.out([f]), clean) for f in faults)
    weak = {k: v for k, v in report.items() if v < MARGIN * thr}
    assert not weak, f"{name}: faults below {MARGIN}x the threshold {thr:g}: {weak}"
