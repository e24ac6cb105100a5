"""Inverse coupling (audio.rs:762-777, steps in reverse at :991-1002): every place the library decouples, the topology
classes each place can take, a numpy restatement of the operation, and the residue columns that give each coupling step
chosen inputs.  Pure Python: the CPU suite checks the restatement against the oracle and that the cases reach every
site with every class; the GPU modules run the cases.

Sites (lewton_b200/csrc; "front stages" = k_floor1_segments + k_prologue_fused, launched once per batch by the paths
below):
  S1  k_prologue_fused<false>, the pipelined loop, nsteps <= 1 (kernel_prologue.cuh:299-306, via d_pf_stereo_quad and
      d_inverse_couple_stereo): the residue entry with 1 or 2 channels and 16-byte aligned arenas;
  S2  the same loop, nsteps >= 2 (kernel_prologue.cuh:307-323): 2 channels, 2 or more steps;
  S3  k_prologue_fused<false>, the general column (kernel_prologue.cuh:362-379): 3-8 channels;
  S4  k_prologue_fused<true>, the serial stereo body (kernel_prologue.cuh:351-358): the VQ entry, <= 2 channels, <= 1 step;
  S5  k_prologue_fused<true>, the general column: the VQ entry, 2 channels with 2 or more steps, or 3-8 channels;
  S6  k_prologue's stereo branch (kernels_generic.cuh:130-143): the four-kernel path (LWB_FORCE_GENERIC=1) on arenas the
      front stages refuse (a residue row off a 16-byte boundary), 2 channels, <= 1 step;
  S7  k_prologue through d_inverse_couple_regs (kernels_generic.cuh:145-159): the same, every other shape of <= 8 channels;
  S8  k_prologue's two passes (kernels_generic.cuh:163-174): more than 8 channels, any path;
  S9  k_chain's front half (kernel_chain.cuh:131-149, d_inverse_couple_regs): interleaved output, <= 8 channels;
  S10 lwb_debug_packet_taps' post_inverse (lwb_api.cu:1224-1238): k_prologue on one packet under unit dense floors.

Which kernels prove a site ran are in SITES; the GPU modules hold every batch to them with expect_kernels.

The dense-residue cases mix floor 1, dense (host floor-0) curves and unused floors within packets; floor-0 records
(LWB_FLOOR_ZERO, curves from k_floor0_curves) are not among them: the oracle's packet stage takes no records."""
import functools

import numpy as np

FLOOR_UNUSED, FLOOR_ONE, FLOOR_DENSE = 0, 1, 2          # lewton_b200.h LWB_FLOOR_*
MAX_COUPLING = 256                                        # LWB_MAX_COUPLING
TINY = np.float32(1.17549435e-38)

# +x -x +0 -0 +inf -inf NaN denormal: test_kernel_edges.CLASSES (the CPU suite keeps the two equal)
CLASSES = np.array([1.5, -2.25, 0.0, -0.0, np.inf, -np.inf, np.nan, 3e-42], np.float32)
PAIRS = [(int(i), int(j)) for i in range(8) for j in range(8)]     # (magnitude class, angle class)
FINITE = (0, 1, 2, 3, 7)

FRONT = frozenset({"k_floor1_segments", "k_prologue_fused"})
# site: (what selects it, kernels that must run, kernels that must not)
SITES = {
    "S1": ("residue entry, C <= 2, <= 1 step, aligned arenas", FRONT, {"k_prologue", "k_chain"}),
    "S2": ("residue entry, C = 2, >= 2 steps, aligned arenas", FRONT, {"k_prologue", "k_chain"}),
    "S3": ("residue entry, 3-8 channels, aligned arenas", FRONT, {"k_prologue", "k_chain"}),
    "S4": ("VQ entry, C <= 2, <= 1 step", FRONT, {"k_prologue", "k_chain"}),
    "S5": ("VQ entry, C = 2 with >= 2 steps or 3-8 channels", FRONT, {"k_prologue", "k_chain"}),
    "S6": ("LWB_FORCE_GENERIC=1, a residue row off 16 bytes, C = 2, <= 1 step", {"k_prologue"}, FRONT | {"k_chain"}),
    "S7": ("LWB_FORCE_GENERIC=1, a residue row off 16 bytes, other shapes of <= 8 channels", {"k_prologue"}, FRONT | {"k_chain"}),
    "S8": ("more than 8 channels", {"k_prologue"}, FRONT | {"k_chain"}),
    "S9": ("interleaved output, <= 8 channels", {"k_chain"}, FRONT | {"k_prologue"}),
    "S10": ("lwb_debug_packet_taps", (), ()),
}


# ---------------------------------------------------------------------------------------------------------------------
# the numpy restatement
# ---------------------------------------------------------------------------------------------------------------------
def inverse_couple(mag, ang):
    """audio.rs:762-777 on f32 arrays, branch for branch; `> 0.` is false for NaN.  Returns (new magnitude, new angle)."""
    m = np.asarray(mag, np.float32)
    a = np.asarray(ang, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        mp, ap = m > 0, a > 0
        nm = np.where(mp, np.where(ap, m, m + a), np.where(ap, m, m - a))
        na = np.where(mp, np.where(ap, m - a, m), np.where(ap, m + a, m))
    return nm.astype(np.float32), na.astype(np.float32)


def decouple(res, coupling, forward=False, exchange=False, record=None):
    """The step loop of audio.rs:991-1002 on res [C][...] (copied): steps in reverse, or forward (forward=True), each
    with magnitude and angle exchanged (exchange=True) -- the last two are what a wrong kernel would do.
    record: a dict that receives {step: (magnitude input, angle input)}."""
    r = np.array(res, np.float32, copy=True)
    order = range(len(coupling)) if forward else range(len(coupling) - 1, -1, -1)
    for s in order:
        m, a = coupling[s]
        if exchange:
            m, a = a, m
        if record is not None:
            record[s] = (r[m].copy(), r[a].copy())
        r[m], r[a] = inverse_couple(r[m], r[a])
    return r


def same_bits(a, b):
    """Element-wise: identical bits, any NaN equal to any NaN."""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def differ_in_bits(a, b):
    return not bool(np.all(np.asarray(a, np.float32).view(np.uint32) == np.asarray(b, np.float32).view(np.uint32)))


def sign_class(x):
    """Index into CLASSES of every element of x."""
    x = np.asarray(x, np.float32)
    neg = np.signbit(x)
    out = np.where(neg, 1, 0)
    out = np.where(x == 0, np.where(neg, 3, 2), out)
    out = np.where((x != 0) & (np.abs(x) < TINY), 7, out)
    out = np.where(np.isinf(x), np.where(neg, 5, 4), out)
    return np.where(np.isnan(x), 6, out)


def step_classes(res, coupling):
    """{step: set of (magnitude class, angle class)} that the reference's step loop feeds each step of res [C][n]."""
    rec = {}
    decouple(res, coupling, record=rec)
    return {s: set(zip(sign_class(m).tolist(), sign_class(a).tolist())) for s, (m, a) in rec.items()}


# ---------------------------------------------------------------------------------------------------------------------
# columns that give each step chosen inputs
# ---------------------------------------------------------------------------------------------------------------------
def free_steps(coupling):
    """Steps that no later step (one the loop runs before it) shares a channel with: their inputs are the raw residue."""
    return [s for s, (m, a) in enumerate(coupling) if not any({m, a} & set(st) for st in coupling[s + 1:])]


@functools.lru_cache(maxsize=None)
def _probe_columns(C, coupling, seed, n_random):
    return probe_columns(C, list(coupling), seed, n_random, cached=False)


def probe_columns(C, coupling, seed=0, n_random=4096, cached=True):
    """{step: {class pair: residue column [C]}}: for each step and (magnitude class, angle class) pair, a column (one bin
    of every channel) whose decoupling by the reference feeds that step that pair.  Candidates: the pair itself on the
    step's channels with the other channels at one of a few fills, then random columns of CLASSES and finite values.
    A step that runs after another one on one of its channels sees that step's outputs, and some pairs are no output of
    a decoupling (say +inf and -inf: m + a and m - a of one (m, a) are not both infinite of opposite signs); such a
    step gets the pairs the candidates reach."""
    if cached:
        return _probe_columns(C, tuple(coupling), seed, n_random)
    S, P = len(coupling), len(PAIRS)
    if not S:
        return {}
    rng = np.random.default_rng(seed)
    v = np.tile(CLASSES[[p[0] for p in PAIRS]], S)
    w = np.tile(CLASSES[[p[1] for p in PAIRS]], S)
    mi = np.repeat([m for m, _ in coupling], P)
    ai = np.repeat([a for _, a in coupling], P)
    cols = np.arange(S * P)
    cands = []
    fills = (np.float32(0), "w", "v", np.float32(-0.0), np.float32(1), np.float32(-1)) if S <= 16 else (np.float32(0),)
    for fill in fills:
        raw = np.empty((C, S * P), np.float32)
        raw[:] = w if isinstance(fill, str) and fill == "w" else v if isinstance(fill, str) else fill
        raw[mi, cols] = v
        raw[ai, cols] = w
        cands.append(raw)
    values = np.concatenate([CLASSES, np.float32([0.75, -3.0, 4.5, -1e-40, 1.5, -2.25])])
    cands.append(rng.choice(values, (C, n_random)).astype(np.float32))
    raw = np.concatenate(cands, axis=1)
    rec = {}
    done = decouple(raw, coupling, record=rec)
    # columns that stay finite from end to end first: a finite pair's column then hides no inf / NaN elsewhere
    order = np.argsort(~(np.isfinite(raw).all(axis=0) & np.isfinite(done).all(axis=0)), kind="stable")
    out = {}
    for s in range(S):
        ids = (sign_class(rec[s][0]) * 8 + sign_class(rec[s][1]))[order]
        u, first = np.unique(ids, return_index=True)
        out[s] = {PAIRS[int(k)]: raw[:, order[i]] for k, i in zip(u, first)}
    return out


def finite_pair(p):
    return p[0] in FINITE and p[1] in FINITE


# ---------------------------------------------------------------------------------------------------------------------
# topology classes
# ---------------------------------------------------------------------------------------------------------------------
def topology(coupling, C):
    """The classes of one mapping's coupling list over C channels."""
    got = set()
    n = len(coupling)
    if n == 0:
        got.add("none")
    elif n == 1:
        got.add("one, magnitude first" if coupling[0][0] < coupling[0][1] else "one, angle first")
    if C == 2 and n >= 2:
        got |= {f"stereo, {k} steps" for k in (2, 3, 8) if n == k}
    if len(set(coupling)) < n:
        got.add("repeated pair")
    if any((a, m) in coupling for m, a in coupling):
        got.add("reversed pair")
    used = [c for st in coupling for c in st]
    if n >= 2 and len(set(used)) < len(used):
        got.add("shared channel")
    if {m for m, _ in coupling} & {a for _, a in coupling}:
        got.add("magnitude and angle")
    if n == MAX_COUPLING:
        got.add(f"{MAX_COUPLING} steps, {'<= 8' if C <= 8 else '> 8'} channels")
    return got


_STEREO_MULTI = {"stereo, 2 steps", "stereo, 3 steps", "stereo, 8 steps", "repeated pair", "reversed pair",
                 "shared channel", "magnitude and angle"}
_ONE = {"one, magnitude first", "one, angle first"}
_COLUMN = {"none"} | _ONE | {"repeated pair", "reversed pair", "shared channel", "magnitude and angle"}
# the classes each site can take
SITE_CLASSES = {
    "S1": {"none"} | _ONE,
    "S2": _STEREO_MULTI,
    "S3": _COLUMN | {f"{MAX_COUPLING} steps, <= 8 channels"},
    "S4": {"none"} | _ONE,
    "S5": _STEREO_MULTI | _COLUMN,
    "S6": {"none"} | _ONE,
    "S7": _STEREO_MULTI | _COLUMN | {f"{MAX_COUPLING} steps, <= 8 channels"},
    "S8": _COLUMN | {f"{MAX_COUPLING} steps, > 8 channels"},
    "S9": _STEREO_MULTI | _COLUMN | {f"{MAX_COUPLING} steps, <= 8 channels"},
    "S10": _STEREO_MULTI | _COLUMN | {f"{MAX_COUPLING} steps, <= 8 channels", f"{MAX_COUPLING} steps, > 8 channels"},
}


def max_steps(rng, C):
    """LWB_MAX_COUPLING random steps over C channels (magnitude != angle)."""
    out = []
    for _ in range(MAX_COUPLING):
        m, a = rng.choice(C, 2, replace=False)
        out.append((int(m), int(a)))
    return out


STEREO = [[], [(0, 1)], [(1, 0)]]
STEREO_MULTI = [[(0, 1), (1, 0)], [(0, 1), (0, 1)], [(1, 0), (0, 1), (1, 0)],
                [(0, 1), (1, 0), (1, 0), (0, 1), (0, 1), (1, 0), (0, 1), (1, 0)]]


def column(C):
    """Mappings of 3 or more channels: none, one step each way, a chain through a shared channel (5.1 style), a channel
    that is magnitude in one step and angle in another, a repeated and a reversed pair."""
    return [[], [(0, C - 1)], [(C - 1, 1)], [(0, 1), (2, 1), (0, 2)], [(1, 2), (0, 1), (2, 0)],
            [(0, 2), (1, 2), (0, 2)], [(C - 1, 0), (0, C - 1), (1, 2)]]


class Case:
    """One batch (or, S10, one set of tap calls): a site, a channel count, the mappings (coupling lists) its setup
    holds, blocksizes, and how it is selected (environment, output format, a misaligned residue arena)."""

    def __init__(self, name, site, C, mappings, bs0=8, bs1=11, env=None, interleaved=False, misalign=False):
        self.name, self.site, self.C, self.mappings = name, site, C, mappings
        self.bs0, self.bs1, self.env, self.interleaved, self.misalign = bs0, bs1, env, interleaved, misalign

    def classes(self):
        return set().union(*(topology(m, self.C) for m in self.mappings))

    def __repr__(self):
        return self.name


GENERIC_ENV = {"LWB_FORCE_GENERIC": "1"}


def cases(seed=4242):
    rng = np.random.default_rng(seed)
    m8, m10 = max_steps(rng, 8), max_steps(rng, 10)
    return [
        Case("S1_mono", "S1", 1, [[]]),
        Case("S1_stereo", "S1", 2, STEREO),
        Case("S2_stereo", "S2", 2, STEREO_MULTI),
        Case("S3_3ch", "S3", 3, column(3)),
        Case("S3_8ch", "S3", 8, column(8) + [m8], bs0=10, bs1=10),      # uniform 1024: k_mid (128/1024 chains go to k_chain)
        Case("S6_stereo", "S6", 2, STEREO, env=GENERIC_ENV, misalign=True),
        Case("S7_mono", "S7", 1, [[]], env=GENERIC_ENV, misalign=True),
        Case("S7_stereo", "S7", 2, STEREO_MULTI, env=GENERIC_ENV, misalign=True),
        Case("S7_8ch", "S7", 8, column(8) + [m8], bs0=7, bs1=10, env=GENERIC_ENV, misalign=True),
        Case("S8_10ch", "S8", 10, column(10) + [m10], bs0=7, bs1=10),
        Case("S9_stereo", "S9", 2, STEREO + STEREO_MULTI, interleaved=True),
        Case("S9_8ch", "S9", 8, column(8) + [m8], bs0=7, bs1=10, interleaved=True),
    ]


def vq_cases():
    """S4, S5: the VQ entry, packer-made streams with these coupling lists (tests/vorbis_packer.py), through the
    four-kernel path, whose front stages are k_floor1_segments + k_prologue_fused<true> on aligned arenas."""
    return [
        Case("S4_mono", "S4", 1, [[]], env=GENERIC_ENV),
        Case("S4_stereo", "S4", 2, STEREO, env=GENERIC_ENV),
        Case("S5_stereo", "S5", 2, STEREO_MULTI, env=GENERIC_ENV),
        Case("S5_6ch", "S5", 6, column(6), env=GENERIC_ENV),
    ]


def tap_cases(seed=4343):
    """S10: one setup per channel count 1..12, every mapping its channel count allows."""
    rng = np.random.default_rng(seed)
    out = []
    for C in range(1, 13):
        maps = [[]] if C == 1 else STEREO + STEREO_MULTI if C == 2 else column(C)
        if C in (8, 12):
            maps = maps + [max_steps(rng, C)]
        out.append(Case(f"S10_{C}ch", "S10", C, maps, bs0=8, bs1=12))
    return out


def reached(case_list):
    """{site: classes} the cases reach."""
    got = {}
    for c in case_list:
        got.setdefault(c.site, set()).update(c.classes())
    return got


# ---------------------------------------------------------------------------------------------------------------------
# packets of a case
# ---------------------------------------------------------------------------------------------------------------------
def mapping_pool(C, coupling):
    """(finite columns, non-finite columns) [C][k] of one mapping.  The finite ones: every column that stays finite in
    every channel through the decoupling (every finite class pair of every step, where its column can); the others: one
    per step (finite_chain / nonfinite_chain lay them out)."""
    probes = probe_columns(C, coupling)
    keys = [(s, p) for s in probes for p in probes[s]]
    cols = np.stack([probes[s][p] for s, p in keys], axis=1) if keys else np.zeros((C, 0), np.float32)
    ok = np.isfinite(cols).all(axis=0) & np.isfinite(decouple(cols, coupling)).all(axis=0)
    ends_finite = dict(zip(keys, ok.tolist()))
    fin = [col for s in probes for p, col in probes[s].items() if ends_finite[s, p]]
    nonfin = [[col for p, col in probes[s].items() if not ends_finite[s, p]] for s in sorted(probes)]
    # round j: step j % S, its (j mod its count)-th non-finite pair: every step one, every pair at some step
    k = max(max((len(x) for x in nonfin), default=0), len(nonfin))
    nf = [nonfin[j % len(nonfin)][j % len(nonfin[j % len(nonfin)])] for j in range(k) if nonfin[j % len(nonfin)]]
    empty = np.zeros((C, 0), np.float32)
    return (np.stack(fin, axis=1) if fin else empty), (np.stack(nf, axis=1) if nf else empty)


def _block(k):
    return 0 if k % 3 == 1 else 1          # a chain's block types: long, short, long, long, short, ...


def finite_chain(rng, C, fin, n0, n1, min_packets=4):
    """[(blockflag, residue [C][n/2])] of a chain that carries every finite probe column of fin (from bin 4 of each
    packet on) among random finite values; n0, n1: n/2 of the short and long blocks.  Every bin of it stays finite
    through the decoupling, so every probe reaches the PCM."""
    out, at = [], 0
    while at < fin.shape[1] or len(out) < min_packets:
        bf = _block(len(out))
        n2 = n1 if bf else n0
        res = (rng.standard_normal((C, n2)) * 0.5).astype(np.float32)
        k = min(n2 - 8, fin.shape[1] - at)
        if k > 0:
            res[:, 4:4 + k] = fin[:, at:at + k]
            at += k
        out.append((bf, res))
    return out


def nonfinite_chain(rng, C, nf, n0, n1):
    """[(blockflag, residue)] of a chain of one packet per non-finite probe column (at bin 1, the other bins random):
    an inf or NaN spreads over its channel's whole block in the IMDCT, and over the next packet's output through the
    overlap, so these packets go in chains of their own, apart from the finite probes."""
    out = []
    for k in range(nf.shape[1]):
        bf = _block(k)
        res = (rng.standard_normal((C, n1 if bf else n0)) * 0.5).astype(np.float32)
        res[:, 1] = nf[:, k]
        out.append((bf, res))
    return out


def floor_kind(j, c, unused=True):
    """The floor kind of channel c of packet j: floor 1 and dense curves alternate over the channels, and (unused) an
    unused floor on one row in six.  The chains of finite probes take none: an unused floor would hide the decoupled
    residue of its channel (0 x residue)."""
    k = (j + c) % 6
    return FLOOR_UNUSED if unused and k == 5 else FLOOR_DENSE if k % 2 else FLOOR_ONE


def window_flags(bf):
    """prev / next window flags of a block-type sequence (short blocks carry none)."""
    n = len(bf)
    prev = np.ones(n, np.uint8)
    nxt = np.ones(n, np.uint8)
    for i in range(n):
        if bf[i]:
            prev[i] = bf[i - 1] if i else 1
            nxt[i] = bf[i + 1] if i + 1 < n else 1
    return prev, nxt


# ---------------------------------------------------------------------------------------------------------------------
# the cross-packet hand-over of the pipelined loop
# ---------------------------------------------------------------------------------------------------------------------
def pf_grid(n_pk, C, sm_count):
    """k_prologue_fused's grid (path_generic.cuh:279): persistent CTAs, CTA b decodes packets b, b + grid, ..."""
    return min(n_pk, sm_count * (4 if C > 2 else 8))


def handover_modes(n_pk, grid, n_modes):
    """Mode index of each packet of a front-stage packet list: packet j + grid gets mode (mode of j) + 3, so that
    consecutive packets of one CTA differ in block size (modes alternate short, long) and mapping (pairs of modes share
    one)."""
    j = np.arange(n_pk)
    return ((j % grid + 3 * (j // grid)) % n_modes).astype(np.uint8)
