"""Host model of the fused MoE decode kernel's schedule (lvllm_b200/csrc/moe_fused.cu), in pure Python.

It replays what every CTA computes in phase 0 (routing table and chunk table) and in the stream-K set-up, and reports for
every (phase, tile) whether it is computed whole or split, by which CTAs and over which k-iterations, the chunk's row
count and whether its last k-iteration loads a single k-block.  ``Schedule.labels`` is the set of kernel branches a launch
reaches; the tests use it to prove that a case exercises what it claims to.

Every rule cites the line of moe_fused.cu (or api.cu / moe_internal.cuh) it restates.  The grid size G is a parameter:
the kernel launches one CTA per SM (moe_fused.cu:1386), so the GPU tests pass ``multi_processor_count``.
"""
from __future__ import annotations

from dataclasses import dataclass, field

# moe_internal.cuh:15, 36-42
ROW_ALIGN = 16
FUSED_MAX_SLOTS = 2048
FUSED_MAX_TOKENS = 256
FUSED_MAX_ROWS = 6144
FUSED_MAX_EXPERTS = 512
FUSED_MAX_CHUNKS = 512
FUSED_MAX_TILES = 65536
FUSED_MAX_J2 = 256

FORMATS = ("bf16", "fp16", "fp8", "fp8_e8m0", "int4", "nvfp4", "mxfp4")
W4 = {"int4": 1, "nvfp4": 2, "mxfp4": 3}


@dataclass(frozen=True)
class Geometry:
    """Layer geometry as make_layer sets it (api.cu:351-371)."""
    fmt: str
    E: int
    H: int
    I: int
    gated: bool = True

    @property
    def wq(self) -> int:
        return W4.get(self.fmt, 0)

    @property
    def fp8(self) -> bool:
        return self.fmt.startswith("fp8")

    @property
    def epk(self) -> int:          # elements per 128-byte k-block (api.cu:366; 4-bit layers have esz_bits 16, :354)
        return 128 if self.fp8 else 64

    @property
    def KB1(self) -> int:
        return self.H // self.epk

    @property
    def KB2(self) -> int:
        return self.I // self.epk

    @property
    def J1(self) -> int:
        return self.I // 128

    @property
    def J2(self) -> int:
        return self.H // 128

    @property
    def w2_paired(self) -> bool:   # api.cu:371
        return self.J2 % 2 == 0

    @property
    def NA(self) -> int:
        return 2 if self.gated else 1


def fused_supported(geo: Geometry, M: int, k: int) -> bool:
    """moe_fused.cu:1403-1414."""
    if geo.wq and not (geo.gated and geo.w2_paired):
        return False
    slots = M * k
    if slots > FUSED_MAX_SLOTS or geo.E > FUSED_MAX_EXPERTS or M > FUSED_MAX_TOKENS:
        return False
    act = min(slots, geo.E)
    if slots + 15 * act > FUSED_MAX_ROWS:
        return False
    chunks = act + slots // 16
    if chunks > FUSED_MAX_CHUNKS:
        return False
    if geo.J2 > FUSED_MAX_J2 or chunks * geo.J1 > FUSED_MAX_TILES or chunks * geo.J2 > FUSED_MAX_TILES:
        return False
    return True


def tn_max(geo: Geometry, M: int) -> int:
    """Chunk width TNMAX: tn / tn4 of moe_fused.cu:1470-1471."""
    if geo.wq:
        return 16 if M <= 16 else 32 if M <= 32 else 64
    return 16 if M <= 16 else 32


def part_start(c: int, n: int, parts: int) -> int:       # moe_fused.cu:176
    return (c * n) // parts


def part_owner(i: int, n: int, parts: int) -> int:       # moe_fused.cu:177-182
    c = (i * parts) // n
    while c + 1 < parts and part_start(c + 1, n, parts) <= i:
        c += 1
    while c > 0 and part_start(c, n, parts) > i:
        c -= 1
    return c


@dataclass(frozen=True)
class Chunk:
    expert: int
    row0: int
    nrows: int
    slots: tuple        # the (token * k + j) slots of the chunk's rows, in row order


def chunk_table(geo: Geometry, ids, tnmax: int):
    """Phase 0a (moe_fused.cu:439-545): stable counting sort of the slots by expert (ids outside [0, E) are skipped,
    :448), every expert's rows padded to ROW_ALIGN (:481, :519), chunks of at most TNMAX rows (:511-518).
    Returns (chunks, row_of_slot)."""
    flat = [int(v) for row in ids for v in row]
    by_e = [[] for _ in range(geo.E)]
    for s, e in enumerate(flat):
        if 0 <= e < geo.E:
            by_e[e].append(s)
    chunks, row_of_slot = [], [-1] * len(flat)
    off = 0
    for e in range(geo.E):
        sl = by_e[e]
        for r, s in enumerate(sl):
            row_of_slot[s] = off + r
        for q in range((len(sl) + tnmax - 1) // tnmax):
            part = tuple(sl[q * tnmax:(q + 1) * tnmax])
            chunks.append(Chunk(e, off + q * tnmax, len(part), part))
        off += (len(sl) + ROW_ALIGN - 1) // ROW_ALIGN * ROW_ALIGN
    return chunks, row_of_slot


@dataclass
class Seg:
    ph: int
    grp: int
    c0: int
    c1: int
    KI: int
    J: int
    N: int
    P: int
    aligned: bool
    ranges: list        # [begin, end) of every CTA


@dataclass
class TileWork:
    """One (phase, tile): the tile is (chunk q, j-th tile of the phase) and spans KI k-iterations."""
    ph: int
    seg: int
    q: int
    j: int
    KI: int
    nrows: int
    parts: list         # (cta, k0, k1) in CTA order
    half: bool          # its last k-iteration loads one k-block (nkb == 1)

    @property
    def split(self) -> bool:
        return len(self.parts) > 1 or self.parts[0][1] != 0 or self.parts[0][2] != self.KI

    @property
    def contributors(self) -> int:
        return len(self.parts)


@dataclass
class Schedule:
    geo: Geometry
    M: int
    k: int
    G: int
    align_g1: int
    supported: bool
    tnmax: int = 0
    chunks: list = field(default_factory=list)
    row_of_slot: list = field(default_factory=list)
    KI1e: int = 0
    KI2: int = 0
    J2e: int = 0
    pair2: bool = True
    NG: int = 0
    segs: list = field(default_factory=list)
    tiles: list = field(default_factory=list)
    labels: set = field(default_factory=set)

    def kblocks(self, ph: int, k0: int, k1: int):
        """The k-blocks (of geo.epk elements) that k-iterations [k0, k1) of a phase-ph tile load (moe_fused.cu:761-762)."""
        geo = self.geo
        KB = geo.KB1 if ph == 0 else geo.KB2
        if self.one_kb_per_iteration(ph):
            return list(range(k0, k1))
        return list(range(2 * k0, min(2 * k1, KB)))

    def one_kb_per_iteration(self, ph: int) -> bool:
        """`two` of moe_fused.cu:751: one k-block of two 128-row tiles per stage, else up to two k-blocks of one tile
        (of one tile pair for the 4-bit formats)."""
        if self.geo.wq:
            return False
        return self.geo.NA == 2 if ph == 0 else self.pair2

    def out_tiles(self, ph: int, j: int):
        """128-row weight tiles (output column tiles of the phase) that schedule tile j of phase ph computes: GEMM1 gate
        (and up) tile j; GEMM2 tiles 2j, 2j + 1 when paired (moe_fused.cu:1268), else j."""
        if ph == 0:
            return [j]
        return [2 * j, 2 * j + 1] if self.pair2 else [j]


def build(geo: Geometry, ids, G: int, align_g1: int = 60) -> Schedule:
    """Replays one launch with the routing `ids` ([M][k] nested sequence or tensor) on a grid of G CTAs."""
    ids = [[int(v) for v in row] for row in (ids.tolist() if hasattr(ids, "tolist") else ids)]
    M, k = len(ids), len(ids[0])
    sch = Schedule(geo, M, k, G, align_g1, fused_supported(geo, M, k))
    if not sch.supported:
        sch.labels.add("grouped_gemm")
        return sch
    lab = sch.labels
    lab.add("fused")
    sch.tnmax = tn_max(geo, M)
    lab.add(f"tnmax{sch.tnmax}")
    sch.chunks, sch.row_of_slot = chunk_table(geo, ids, sch.tnmax)
    n_chunks = len(sch.chunks)
    if n_chunks == 0:
        lab.add("no_rows")            # moe_fused.cu:548-562: the output is zero-filled, no GEMM runs
        return sch
    wd = geo.wq != 0
    # moe_fused.cu:686-690
    sch.KI1e = geo.KB1 if (geo.NA == 2 and not wd) else (geo.KB1 + 1) // 2
    sch.pair2 = geo.w2_paired
    sch.KI2 = geo.KB2 if (sch.pair2 and not wd) else (geo.KB2 + 1) // 2
    sch.J2e = geo.J2 // 2 if sch.pair2 else geo.J2
    sch.NG = 2 if n_chunks >= 4 else 1
    lab.add(f"ng{sch.NG}")
    lab.add("g2_paired" if sch.pair2 else "g2_unpaired")
    # moe_fused.cu:693-725
    split_at = n_chunks // 2 if sch.NG == 2 else n_chunks
    for ph in range(2):
        for g in range(sch.NG):
            c0 = 0 if g == 0 else split_at
            c1 = n_chunks if g == sch.NG - 1 else split_at
            KI = sch.KI1e if ph == 0 else sch.KI2
            J = geo.J1 if ph == 0 else sch.J2e
            N = (c1 - c0) * J * KI
            P = min(N, G)
            n_tiles = (c1 - c0) * J
            waves = (n_tiles + G - 1) // G
            aligned = ((ph == 1 and n_tiles * 10 >= waves * G * 7) or
                       (ph == 0 and align_g1 > 0 and waves <= 3 and n_tiles * 100 >= waves * G * align_g1))
            if aligned:
                P = G
                ranges = [(part_start(c, n_tiles, G) * KI, part_start(c + 1, n_tiles, G) * KI) for c in range(G)]
            else:
                ranges = [(part_start(c, N, P), part_start(c + 1, N, P)) if c < P else (0, 0) for c in range(G)]
            sch.segs.append(Seg(ph, g, c0, c1, KI, J, N, P, aligned, ranges))
            lab.add(f"g{ph + 1}_{'aligned' if aligned else 'streamk'}")
    # tiles and their contributors (the drain / fix-up loops, moe_fused.cu:907-911, 1090-1097)
    for si, sg in enumerate(sch.segs):
        parts = {}
        for cta, (b, e) in enumerate(sg.ranges):
            it = b
            while it < e:
                tile, k0 = divmod(it, sg.KI)
                k1 = sg.KI if sg.KI - k0 < e - it else k0 + (e - it)
                parts.setdefault(tile, []).append((cta, k0, k1))
                it += k1 - k0
        KB = geo.KB1 if sg.ph == 0 else geo.KB2
        half = (not sch.one_kb_per_iteration(sg.ph)) and KB % 2 == 1
        for tile in sorted(parts):
            q = sg.c0 + tile // sg.J
            sch.tiles.append(TileWork(sg.ph, si, q, tile % sg.J, sg.KI, sch.chunks[q].nrows, parts[tile], half))
    fb = 8 if wd else 16               # moe_fused.cu:1125
    for t in sch.tiles:
        p = f"g{t.ph + 1}"
        if t.half:
            lab.add(f"{p}_half_iter")
        if not t.split:
            lab.add(f"{p}_whole")
            if t.ph == 1:
                continue               # straight to y from the drain warps (moe_fused.cu:983-1023)
        else:
            lab.add(f"{p}_split")
            if t.nrows <= 4:           # one round trip per 16 contributors (moe_fused.cu:1145-1171)
                lab.add(f"{p}_fix_small")
                if t.contributors > 16:
                    lab.add(f"{p}_fix_small_multi")
            else:                      # rounds of 4 contributors (moe_fused.cu:1172-1197)
                lab.add(f"{p}_fix_wide")
                if t.contributors > 16:
                    lab.add(f"{p}_fix_wide_gt16")
                if t.nrows <= 16:
                    lab.add(f"{p}_split_rows5_16")
                else:
                    lab.add(f"{p}_split_rows17_32" if t.nrows <= 32 else f"{p}_split_rows33_64")
        nblk = (t.nrows + fb - 1) // fb   # finalisation blocks of FB token columns (moe_fused.cu:1136)
        if wd and nblk == 8:
            lab.add("w4_fix_8blocks")
    return sch


def check_invariants(sch: Schedule) -> None:
    """The properties the kernel's cross-CTA protocol relies on; raises AssertionError."""
    geo = sch.geo
    if sch.supported:
        assert len(sch.chunks) <= FUSED_MAX_CHUNKS, "chunk table overflow while fused_supported holds"
        rows = sum((n + ROW_ALIGN - 1) // ROW_ALIGN * ROW_ALIGN for n in
                   _expert_counts(sch).values())
        assert rows <= FUSED_MAX_ROWS
    for si, sg in enumerate(sch.segs):
        # every (tile, k-iteration) exactly once
        cover = [0] * sg.N
        for b, e in sg.ranges:
            for i in range(b, e):
                cover[i] += 1
        assert all(c == 1 for c in cover), f"segment {si}: coverage {set(cover)}"
    for t in sch.tiles:
        sg = sch.segs[t.seg]
        assert [p[0] for p in t.parts] == list(range(t.parts[0][0], t.parts[-1][0] + 1)), "contributors not contiguous"
        assert t.parts[0][1] == 0 and t.parts[-1][2] == t.KI
        for a, b in zip(t.parts, t.parts[1:]):
            assert a[2] == b[1]
        if t.split:
            base = (t.q - sg.c0) * sg.J + t.j
            cf = part_owner(base * sg.KI, sg.N, sg.P)
            cl = part_owner(base * sg.KI + sg.KI - 1, sg.N, sg.P)
            # cf owns k = 0 and [cf, cl] are exactly the contributors (moe_fused.cu:1107-1109)
            assert cf == t.parts[0][0] and cl == t.parts[-1][0], (cf, cl, t.parts)
            assert not sg.aligned
    # per CTA and segment at most one split part starts at k = 0 and at most one at k != 0: the partials slot is
    # (seg * G + cta) * 2 + (k0 != 0 ? 0 : 1) (moe_fused.cu:1027) and the reader picks (cc == cf ? 1 : 0) (:1160, :1186)
    seen = {}
    for t in sch.tiles:
        if not t.split:
            continue
        for cta, k0, _ in t.parts:
            key = (t.seg, cta, k0 != 0)
            assert key not in seen, f"partials slot {key} written twice"
            seen[key] = t


def _expert_counts(sch: Schedule):
    c = {}
    for ch in sch.chunks:
        c[ch.expert] = c.get(ch.expert, 0) + ch.nrows
    return c
