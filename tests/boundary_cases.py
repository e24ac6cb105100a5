"""Where a long-block run of the fused synthesis kernels meets its neighbours: the boundary sites, a plan model that says
which sites a batch reaches and which launches it makes, and case builders that force every site.

The bodies (kernel_long.cuh, kernel_short.cuh):
  * out_block<FIRST>: packet 0 of a long-block run, from a state row, a boundary slot or no history;
  * out_first_short: packet 0 of a long-block run after a short block (first_short 1: read the state; 2: export the
    windowed left slope to a boundary slot for the short block's kernel);
  * end_of_run<LS>: a run's end -- store_right_half, nothing (a cut piece before the last), or the last_short tail:
    x[1024, 1024 + ls) emitted (unless nothing was, one packet without history) and the pl samples behind them kept;
  * short_tail: a short run that completes the boundary slot a long run exported (k_short, k_short_g).

An off-by-one in these bodies corrupts only the samples next to a window transition, so every site below is a row the
GPU tests decode against the oracle.  SITES names each one by kernel, body and flag class; `Plan` restates the
host planner (path_mixed.cuh, path_generic.cuh) closely enough to say, from a batch, which sites each kernel receives
and how often each kernel is launched.  The GPU tests hold the real planner to the launch counts, which ties the model
to it; the CPU tests hold the model's walk to the oracle's overlap rules and the cases to every site.
"""
import re
from collections import Counter, namedtuple

import numpy as np

LONG_N2, SHORT_N, SHORT_N2 = 1024, 256, 128
LS256 = (2048 - 256) // 4          # kernel_long.cuh kLongLs256: the compile-time LS of k_long_s
LONG_WARPS = SHORT_WARPS = 8       # LWB_LONG_WARPS, LWB_SHORT_WARPS
SHORT_OCT = 8                      # kShortOct
OK, BAD_FORMAT, MISMATCH = 0, 1, 3  # LWB_OK, LWB_ERR_BAD_FORMAT, LWB_ERR_MISMATCH
RUNTIME_LS_BS0 = (6, 7, 8, 9, 10)   # blocksize_0 of k_long's runtime-ls transitions (bs1 = 11)

SYNTH_KERNELS = ("k_long", "k_long_s", "k_mid", "k_short", "k_short_g", "k_row_copy", "k_chain")

# ---------------------------------------------------------------------------------------------------------------------
# the site table: id -> (kernel, body, flag class)
# ---------------------------------------------------------------------------------------------------------------------
Site = namedtuple("Site", "kernel body flags")
SITES = {
    # k_long_s: the one pass (round 0), ls = 448 at compile time
    "L1": Site("k_long_s", "out_block<FIRST>", "has_prev: packet 0 overlaps a state row or a pre-copy slot"),
    "L2": Site("k_long_s", "out_block<FIRST>", "piece 0 without history: packet 0 emits nothing"),
    "L3": Site("k_long_s", "out_block<FIRST>", "cut piece k > 0: a primer packet, has_prev 0"),
    "L4": Site("k_long_s", "out_first_short", "first_short 1 with history: reads its state (row or pre-copy slot)"),
    "L5": Site("k_long_s", "out_first_short", "first_short 2: exports the left slope to a boundary slot"),
    "L6": Site("k_long_s", "out_first_short", "first_short 1 without history: nothing emitted"),
    "L7": Site("k_long_s", "end_of_run", "write_state, not last_short: store_right_half to the state row"),
    "L8": Site("k_long_s", "end_of_run", "write_state 0 (a cut piece before the last): nothing stored"),
    "L9": Site("k_long_s", "end_of_run<448>", "last_short, emitted, kept in a boundary slot"),
    "L10": Site("k_long_s", "end_of_run<448>", "last_short, emitted, kept in the state row (the chain ends before a short block)"),
    "L11": Site("k_long_s", "end_of_run<448>", "last_short, one packet without history: kept, nothing emitted"),
    "L12": Site("k_long_s", "end_of_run<448>", "last_short on a cut piece k > 0 (has_prev 0, npk > 1: emitted)"),
    "L13": Site("k_long_s", "cut_run", "a cut segment whose piece 0 is first_short and whose last piece is last_short"),
    # k_long: the rounds, ls passed at run time
    "K1": Site("k_long", "out_block<FIRST>", "has_prev: packet 0 overlaps the state row"),
    "K2": Site("k_long", "out_block<FIRST>", "piece 0 without history: packet 0 emits nothing"),
    "K3": Site("k_long", "out_block<FIRST>", "cut piece k > 0: a primer packet, has_prev 0"),
    "K4": Site("k_long", "out_first_short", "first_short 1 without history: nothing emitted"),
    "K5": Site("k_long", "end_of_run", "write_state, not last_short: store_right_half"),
    "K6": Site("k_long", "end_of_run", "write_state 0 (a cut piece before the last): nothing stored"),
    "K7": Site("k_long", "end_of_run<0>", "last_short, one packet without history: kept, nothing emitted"),
    "K8": Site("k_long", "end_of_run<0>", "last_short on a cut piece k > 0 (has_prev 0, npk > 1: emitted)"),
    "K9": Site("k_long", "cut_run", "a cut segment whose piece 0 is first_short and whose last piece is last_short"),
    # k_short: runs of full-window 256-point blocks
    "S1": Site("k_short", "packet 0", "has_prev: overlaps a state row, a boundary slot or a pre-copy slot"),
    "S2": Site("k_short", "packet 0", "without history: emits nothing (koff 1)"),
    "S3": Site("k_short", "short_tail", "tail after a run with history (out + 128 npk)"),
    "S4": Site("k_short", "short_tail", "tail after a run without history (out + 128 (npk - 1))"),
    "S5": Site("k_short", "short_tail", "tail on cut piece k > 0 of a segment of 32 packets or more"),
    "S6": Site("k_short", "end of run", "a cut piece before the last: neither state nor tail"),
    "S7": Site("k_short", "store_end_state_s", "write_state: the end state to the state row"),
    # k_short_g: bursts of fewer than eight short blocks in the pass, eight runs of one length per warp
    "S8": Site("k_short_g", "short_tail", "burst with history, tail (out + 128 npk)"),
    "S9": Site("k_short_g", "short_tail", "burst on an empty stream, tail (out + 128 (npk - 1))"),
    "S10": Site("k_short_g", "store_end_state_s", "burst with write_state: the end state to the state row"),
    "S11": Site("k_short_g", "group", "dummy positions of a group padded to eight runs"),
    # routing and hand-over (MixedSchedule::plan, segment_chain)
    "R1": Site("k_row_copy", "pre-copy", "pass chain whose first segment is long after long with history: 8 slots per channel"),
    "R2": Site("k_row_copy", "pre-copy", "pass chain whose first segment is long after short with history: 1 slot"),
    "R3": Site("k_row_copy", "pre-copy", "pass chain whose first segment is short with history: 1 slot"),
    "R4": Site("k_long_s", "pass", "a single-segment chain in the pass: its state row read and written in place"),
    "R5": Site("k_long_s", "pass", "first_short 2 runs beside first_short 1 runs in one launch"),
    "R6": Site("k_long", "rounds", "k_long_s (round 0) and k_long (later rounds) in one batch"),
    "R7": Site("k_long", "segment_chain", "long (prev flag 0) after long (next flag 0): two adjacent long segments, rounds"),
    "R8": Site("k_chain", "segment_chain", "long with prev flag 1 on a pl-sample state: the chain kernel"),
}
# k_long's transitions with ls at run time, per blocksize_0: out_first_short with history (F) and the last_short end of
# run, emitted and kept (E).  ls = (2048 - 2^bs0) / 4, pl = 1024 - 2 ls; at bs0 = 8 they meet k_long_s's LS = 448.
for _b in RUNTIME_LS_BS0:
    _ls = (2048 - (1 << _b)) // 4
    SITES[f"T{_b}F"] = Site("k_long", "out_first_short", f"first_short 1 with history, ls {_ls}, pl {1024 - 2 * _ls}")
    SITES[f"T{_b}E"] = Site("k_long", "end_of_run<0>", f"last_short, emitted and kept, ls {_ls}, pl {1024 - 2 * _ls}")


# ---------------------------------------------------------------------------------------------------------------------
# the plan model
# ---------------------------------------------------------------------------------------------------------------------
Geom = namedtuple("Geom", "n ls le rs re blockflag slope_sel")


def geometry(bs0, bs1, bf, pf, nf):
    """host_objects.cuh geometry() (audio.rs:1056-1073): a short block ignores its flags."""
    n, n0 = 1 << (bs1 if bf else bs0), 1 << bs0
    prev, nxt = (pf != 0, nf != 0) if bf else (True, True)
    ls, le, sel = (0, n >> 1, bool(bf)) if prev else ((n - n0) >> 2, (n + n0) >> 2, False)
    rs, re_ = (n >> 1, n) if nxt else ((3 * n - n0) >> 2, (3 * n + n0) >> 2)
    return Geom(n, ls, le, rs, re_, bool(bf), sel)


Walk = namedtuple("Walk", "packets status end samples")    # packets: [(k, geom, has, plen)]; end: (has, plen)


def walk(bs0, bs1, state, bf, pf, nf):
    """path_generic.cuh walk_chain(): the packets a chain decodes from stream state (has, plen), each with the state
    entering it; a slope shorter than the state stops with BAD_FORMAT and empties the state, ls + plen > n stops with
    MISMATCH and keeps it."""
    has, plen = state
    out, pos, status = [], 0, OK
    for k in range(len(bf)):
        g = geometry(bs0, bs1, bf[k], pf[k], nf[k])
        if has:
            if (1 << ((bs1 if g.slope_sel else bs0) - 1)) < plen:
                return Walk(out, BAD_FORMAT, (False, 0), pos)
            if g.ls + plen > g.n:
                return Walk(out, MISMATCH, (has, plen), pos)
        out.append((k, g, has, plen))
        if has:
            pos += g.rs - g.ls
        has, plen = True, g.re - g.rs
    return Walk(out, status, (has, plen), pos)


SEG_CHAIN, SEG_LONG, SEG_SHORT = "chain", "long", "short"
Seg = namedtuple("Seg", "kind first_short last_short p0 n has plen")


def segment(bs0, w, no_short=False):
    """path_mixed.cuh segment_chain(): maximal runs of long blocks (k_long), of full-window 256-point blocks (k_short)
    and of the rest (k_chain); a long run ends at a block before a short one and starts at one after a short one."""
    pl_short = 1 << (bs0 - 1)
    pk = []
    for k, g, has, plen in w.packets:
        kind, fs, lsh = SEG_CHAIN, False, False
        if g.blockflag and g.n == 2048:
            fs = g.ls != 0
            if not has or plen == (pl_short if fs else LONG_N2):
                kind, lsh = SEG_LONG, g.re != g.n
        elif (g.n == SHORT_N and bs0 == 8 and not no_short and g.ls == 0 and g.rs == SHORT_N2 and g.re == SHORT_N
              and (not has or plen == SHORT_N2)):
            kind = SEG_SHORT
        pk.append(Seg(kind, fs if kind == SEG_LONG else False, lsh, k, 1, has, plen))
    segs, k = [], 0
    while k < len(pk):
        j = k + 1
        while j < len(pk) and pk[j].kind == pk[k].kind and not (pk[k].kind == SEG_LONG and (pk[j - 1].last_short or pk[j].first_short)):
            j += 1
        segs.append(pk[k]._replace(n=j - k, last_short=pk[j - 1].last_short))
        k = j
    return segs


def cut_run(n, cuts, has):
    """path_generic.cuh cut_run(): pieces (k, packets, has_prev, write_state); piece k > 0 re-transforms a primer."""
    out = []
    for k in range(cuts):
        p0, p1 = n * k // cuts, n * (k + 1) // cuts
        out.append((k, p1 - p0 if k == 0 else p1 - p0 + 1, has if k == 0 else False, k + 1 == cuts))
    return out


LongPiece = namedtuple("LongPiece", "kernel chain seg k cuts npk has_prev write_state first_short last_short to_slot ls")
ShortPiece = namedtuple("ShortPiece", "kernel chain seg k cuts npk has_prev write_state tail")


class Plan:
    """What one batch does: per chain its walk and segments, whether it takes the pass, the run pieces each kernel
    receives, the launches per kernel and the sites reached."""

    def __init__(self, setup, chains, sm, env=None, memory="device"):
        """setup: (C, bs0, bs1); chains: [(state (has, plen), bf, pf, nf)]; sm: the device's SM count; env: the test
        switches set (LWB_MIXED_ROUNDS, LWB_NO_BURSTS, LWB_NO_SHORT, LWB_E2E_CHUNKS, LWB_NO_MIXED); memory: "device" or
        "host"."""
        env = env or {}
        C, bs0, bs1 = setup
        self.C, self.bs0 = C, bs0
        self.walks = [walk(bs0, bs1, st, bf, pf, nf) for st, bf, pf, nf in chains]
        self.launches = Counter({k: 0 for k in SYNTH_KERNELS})
        self.long, self.short, self.sites = [], [], set()
        self.dummies = 0
        self.path = self._path(chains, env, bs1)
        if self.path != "mixed":
            if self.path == "chain":
                self.launches["k_chain"] = 1
            return
        ls_long = (2048 - (1 << bs0)) >> 2
        self.segs = [segment(bs0, w, "LWB_NO_SHORT" in env) for w in self.walks]
        self._plan(enabled="LWB_MIXED_ROUNDS" not in env and ls_long == LS256, bursts="LWB_NO_BURSTS" not in env)
        if not self.max_rounds:
            return
        n = len(chains)
        n_chunks = 1
        if memory == "host":
            n_chunks = max(1, min(int(env["LWB_E2E_CHUNKS"]), min(64, n))) if "LWB_E2E_CHUNKS" in env else 1
        for kc in range(n_chunks):
            self._chunk(range(n * kc // n_chunks, n * (kc + 1) // n_chunks), sm, ls_long)
        self._piece_sites()
        self._route_sites()

    # lwb_api.cu kBatchPaths: try_long takes uniform long batches; try_mixed those mixed_shape accepts
    def _path(self, chains, env, bs1):
        if "LWB_NO_MIXED" in env:
            return "chain"
        if bs1 == 11 and all(not st[0] or st[1] == LONG_N2 for st, *_ in chains) and all(
                len(w.packets) == len(c[1]) and all(g.blockflag and pf and nf for (_, g, _, _), pf, nf in zip(w.packets, c[2], c[3]))
                for w, c in zip(self.walks, chains)):
            return "long"
        fast = total = 0
        for st, bf, pf, nf in chains:       # mixed_shape(): half the packets or more for the fused kernels
            total += len(bf)
            fast += sum(1 for b in bf if (b and bs1 == 11) or (not b and self.bs0 == 8 and "LWB_NO_SHORT" not in env))
        assert bs1 == 11 and fast * 2 >= total, "the model covers the segmented path's batches only"
        return "mixed"

    def _plan(self, enabled, bursts):
        """MixedSchedule::plan (path_mixed.cuh:117-152), needs_precopy and pre_units (:109-111)."""
        self.max_rounds = max([len(s) for s in self.segs] + [0])
        self.pass_ = [False] * len(self.segs)
        self.round_base, self.bursts = 0, False
        rest = pk_pass = pk_all = 0
        for i, segs in enumerate(self.segs):
            ok = enabled and self.max_rounds > 1 and len(segs) > 0
            for q, sg in enumerate(segs):
                if not ok:
                    break
                if sg.kind == SEG_CHAIN or (q and sg.kind == segs[q - 1].kind):
                    ok = False
                elif sg.kind == SEG_LONG and ((q and not sg.first_short) or (q + 1 < len(segs) and not sg.last_short)):
                    ok = False
            self.pass_[i] = ok
            if ok:
                pk_pass += len(self.walks[i].packets)
            else:
                rest = max(rest, len(segs))
            pk_all += len(self.walks[i].packets)
        if not pk_pass or pk_pass * 2 < pk_all:
            self.pass_ = [False] * len(self.segs)
            return
        self.round_base, self.max_rounds, self.bursts = 1, 1 + rest, bursts

    def needs_precopy(self, i):
        return self.pass_[i] and len(self.segs[i]) > 1 and self.segs[i][0].has

    def pre_units(self, i):
        s0 = self.segs[i][0]
        return LONG_N2 // SHORT_N2 if s0.kind == SEG_LONG and not s0.first_short else 1

    def round_of(self, i, q):
        return 0 if self.pass_[i] else self.round_base + q

    def round_segs(self, i, r):
        n = len(self.segs[i])
        if self.pass_[i]:
            return range(0, n if r == 0 else 0)
        q = n if r < self.round_base else min(r - self.round_base, n)
        return range(q, min(q + 1, n))

    def _chunk(self, idx, sm, ls_long):
        """mixed_layout's round cuts (path_mixed.cuh:218-238), MixedChunk::cuts (:202-207), and MixedWriter's long_seg,
        short_seg and round (:299-387) for the chains idx of one chunk."""
        R, C = self.max_rounds, self.C
        target, target_s = sm * LONG_WARPS * 2, sm * SHORT_WARPS * 2
        rl, rs = [0] * R, [0] * R
        for i in idx:
            for q, sg in enumerate(self.segs[i]):
                if sg.kind != SEG_CHAIN:
                    (rl if sg.kind == SEG_LONG else rs)[self.round_of(i, q)] += C
        cut_l = [min(16, -(-target // v)) if v and v < target else 1 for v in rl]
        cut_s = [min(64, -(-target_s // v)) if v and v < target_s else 1 for v in rs]
        for r in range(R):
            nr = ns = nc = nx = 0
            bursts = []
            kernel = "k_long_s" if self.round_base and r == 0 else "k_long"
            fs_seen = set()
            for i in idx:
                for q in self.round_segs(i, r):
                    sg, nseg = self.segs[i][q], len(self.segs[i])
                    more = self.pass_[i] and q + 1 < nseg
                    if sg.kind == SEG_LONG:
                        cuts = max(1, min(cut_l[r], sg.n // 6))          # kMinCutRun
                        for k, npk, hp, ws in cut_run(sg.n, cuts, sg.has):
                            p = LongPiece(kernel, i, q, k, cuts, npk, hp, ws,
                                          (2 if self.pass_[i] and q else int(sg.first_short)) if k == 0 else 0,
                                          sg.last_short and k + 1 == cuts, more and k + 1 == cuts, ls_long)
                            self.long.append(p)
                            fs_seen.add(p.first_short)
                        nr += C * cuts
                        if q == 0 and self.needs_precopy(i):
                            nx += C
                    elif sg.kind == SEG_SHORT:
                        burst = self.bursts and self.pass_[i] and sg.n < SHORT_OCT
                        cuts = max(1, min(cut_s[r], sg.n // 16))        # kMinCutShort
                        for k, npk, hp, ws in cut_run(sg.n, cuts, sg.has):
                            last = k + 1 == cuts
                            p = ShortPiece("k_short_g" if burst else "k_short", i, q, k, cuts, npk, hp, ws and not (last and more), last and more)
                            self.short.append(p)
                            if burst:
                                bursts += [npk] * C          # one run per channel
                        if not burst:
                            ns += C * cuts
                        if q == 0 and self.needs_precopy(i):
                            nx += C
                    else:
                        nc += 1
            groups = sum(-(-n // SHORT_OCT) for n in Counter(bursts).values())     # group_runs(): per length, padded to 8
            self.dummies += groups * SHORT_OCT - len(bursts)
            for name, cnt in (("k_row_copy", nx), (kernel, nr), ("k_short", ns), ("k_short_g", groups), ("k_chain", nc)):
                if cnt:
                    self.launches[name] += 1
            if kernel == "k_long_s" and {1, 2} <= fs_seen:
                self.sites.add("R5")

    def _piece_sites(self):
        self.sites |= {s for p in self.long for s in long_sites(p, self.bs0)}
        self.sites |= {s for p in self.short for s in short_sites(p)}
        if self.dummies:
            self.sites.add("S11")
        segs_fs_ls = {(p.chain, p.seg) for p in self.long if p.k == 0 and p.first_short and p.cuts > 1}
        for p in self.long:
            if p.last_short and p.k > 0 and (p.chain, p.seg) in segs_fs_ls:
                self.sites.add("L13" if p.kernel == "k_long_s" else "K9")
        if self.launches["k_long_s"] and self.launches["k_long"]:
            self.sites.add("R6")

    def _route_sites(self):
        for i, segs in enumerate(self.segs):
            if self.needs_precopy(i):
                s0 = segs[0]
                self.sites.add("R1" if self.pre_units(i) > 1 else "R2" if s0.kind == SEG_LONG else "R3")
            if self.pass_[i] and len(segs) == 1:
                self.sites.add("R4")
            for q in range(1, len(segs)):
                if segs[q].kind == SEG_LONG and segs[q - 1].kind == SEG_LONG:
                    self.sites.add("R7")
            for k, g, has, plen in self.walks[i].packets:
                if g.n == 2048 and has and g.ls == 0 and plen != LONG_N2:
                    self.sites.add("R8")


def long_sites(p, bs0):
    """The sites a k_long / k_long_s run piece reaches (out_block / out_first_short at packet 0, end_of_run)."""
    s = set()
    pass_ = p.kernel == "k_long_s"
    b = bs0
    if p.k > 0:
        s.add("L3" if pass_ else "K3")
    elif p.first_short == 2:
        s.add("L5")
    elif p.first_short == 1:
        if p.has_prev:
            s.add("L4" if pass_ else f"T{b}F")
        else:
            s.add("L6" if pass_ else "K4")
    else:
        s.add(("L1" if pass_ else "K1") if p.has_prev else ("L2" if pass_ else "K2"))
    if p.last_short:
        emitted = p.npk > 1 or p.has_prev            # end_of_run(): kernel_long.cuh:829-830 (no dummy in these kernels)
        if not emitted:
            s.add("L11" if pass_ else "K7")
        elif pass_:
            s.add("L9" if p.to_slot else "L10")
        else:
            s.add(f"T{b}E")
        if p.k > 0:
            s.add("L12" if pass_ else "K8")
    else:
        s.add(("L7" if pass_ else "K5") if p.write_state else ("L8" if pass_ else "K6"))
    return s


def short_sites(p):
    """The sites a k_short / k_short_g run piece reaches."""
    s = set()
    if p.kernel == "k_short":
        if p.k == 0:
            s.add("S1" if p.has_prev else "S2")
        if p.tail:
            s.add("S5" if p.k > 0 else "S3" if p.has_prev else "S4")
        elif p.write_state:
            s.add("S7")
        else:
            s.add("S6")
    else:
        if p.tail:
            s.add("S8" if p.has_prev else "S9")
        if p.write_state:
            s.add("S10")
    return s


# ---------------------------------------------------------------------------------------------------------------------
# case builders
# ---------------------------------------------------------------------------------------------------------------------
_TOKEN = re.compile(r"S|L[01]{2}|L|\|")


def stream(text):
    """A stream written as packets: S (short), L (long, flags from its neighbours) or Lpn (long with explicit previous
    and next window flags p, n), batches separated by |.  Returns [(bf, pf, nf)] per batch, flags consistent across
    the batch boundaries where not explicit."""
    toks = [t for t in _TOKEN.findall(text.replace(" ", ""))]
    pk = [t for t in toks if t != "|"]
    bf = [0 if t == "S" else 1 for t in pk]
    pf, nf = [], []
    for i, t in enumerate(pk):
        if len(t) == 3:
            pf.append(int(t[1])), nf.append(int(t[2]))
        elif t == "L":
            pf.append(bf[i - 1] if i else 1), nf.append(bf[i + 1] if i + 1 < len(pk) else 1)
        else:
            pf.append(1), nf.append(1)
    out, cur, i = [], ([], [], []), 0
    for t in toks + ["|"]:
        if t == "|":
            out.append(tuple(np.array(a, np.uint8) for a in cur))
            cur = ([], [], [])
        else:
            for a, v in zip(cur, (bf[i], pf[i], nf[i])):
                a.append(v)
            i += 1
    return out


Case = namedtuple("Case", "name bs0 C streams why")


def case(name, streams, why, bs0=8, C=2):
    """streams: stream() texts with the same number of batches; the last batch continues every stream."""
    parsed = [stream(t) for t in streams]
    assert len({len(p) for p in parsed}) == 1 and all(len(b[0]) for p in parsed for b in p), name
    return Case(name, bs0, C, parsed, why)


def n_batches(c):
    return len(c.streams[0])


def plans(c, sm, env=None, memory="device"):
    """The Plan of every batch of case c, stream states carried from batch to batch."""
    states = [(False, 0)] * len(c.streams)
    out = []
    for b in range(n_batches(c)):
        p = Plan((c.C, c.bs0, 11), [(states[s],) + c.streams[s][b] for s in range(len(c.streams))], sm, env, memory)
        out.append(p)
        states = [w.end for w in p.walks]
    return out


def case_sites(c, sm, env=None, memory="device"):
    return set().union(*(p.sites for p in plans(c, sm, env, memory)))


L24 = "L" * 24
CASES = {c.name: c for c in [
    case("precopy", [
        "L L L | L L S S L L | S L L",            # first segment long after long with history: 8-slot pre-copy
        "L S | L L S L L L S | L S",              # long after short with history (first_short 1) beside first_short 2
        "S S | S S L L | S S L",                  # first segment short with history
        "L S S | L L L L | S L",                  # one segment: the state row in place
        "L L | L L L | L S",                      # one long segment ending before a long block: store_right_half
    ], "R1-R5: each kind of pre-copy, a single-segment chain, and first_short 1 and 2 in one k_long_s launch"),
    case("empty_streams", [
        "L L S S L L | L S L",                    # a run without history, emitted at its last_short end
        "L S L L | S L",                          # one long packet without history before a short one: kept, not emitted
        "S S L L | S S L",                        # a burst on an empty stream completes a slot (npk - 1)
        "L00 S L L | S L",                        # first_short without history
        "S L S S S S S S S S L | L S",            # a lone short packet without history, then eight short blocks
    ], "L2, L6, L11, S2, S4, S9: every body on a stream without history"),
    case("cuts", [
        "L S | S " + "L" * 30 + " S S L | S L",    # a cut long segment behind a short one: first_short 2 ... last_short
        "L S | " + L24 + " S L | S L",            # a cut first segment after a short block: first_short 1 ... last_short
        "L S | " + "S" * 40 + " L L | S L",        # a cut short segment of 40 packets whose last piece has the tail
        "L L | L L S L | L L",
    ], "L3, L8, L12, L13, S5, S6: cut pieces and the ends of cut segments, short and long"),
    case("rounds_beside_pass", [
        "L S | L L10 L01 L S S L | S L",          # two adjacent long segments (inconsistent flags): rounds
        "L S | L11 L S S L | S L",                # a long block with prev flag 1 on a 128-sample state: k_chain
        "L S | L S L L S L L S L | S L",          # pass chains beside them, more packets than the rest
        "S S | S L L S L L L S S | L S",
        "L S | L L S L L S L L S | S L",
    ], "R6, R7, R8: chains outside the pass run their rounds (k_long, k_short, k_chain) behind k_long_s"),
]}
# k_long's runtime ls: blocksize_0 6-10 (at 8 also the one pass)
for _b in RUNTIME_LS_BS0:
    CASES[f"runtime_ls_{_b}"] = case(f"runtime_ls_{_b}", [
        "L L S | L L S L L L S L L | S L L",
        "L S | L L L S L L S L | L L S",
        "L L | L S L L L L | L S",
    ], f"T{_b}F, T{_b}E: k_long's transitions with ls = {(2048 - (1 << _b)) // 4} passed at run time", bs0=_b)

# the test switches a row may set, and the sites each (case, switch) row exists for
ROUNDS, NO_BURSTS, CHUNKS = {"LWB_MIXED_ROUNDS": "1"}, {"LWB_NO_BURSTS": "1"}, {"LWB_E2E_CHUNKS": "3"}
Row = namedtuple("Row", "case env sites")
ROWS = [
    Row("precopy", None, {"R1", "R2", "R3", "R4", "R5", "L1", "L4", "L5", "L7", "L9", "L10", "S8", "S10", "S11"}),
    Row("precopy", ROUNDS, {"K1", "K5", "T8F", "T8E", "S1", "S7"}),
    Row("precopy", NO_BURSTS, {"S1", "S3", "S7"}),
    Row("empty_streams", None, {"L2", "L6", "L11", "S9"}),
    Row("empty_streams", ROUNDS, {"K2", "K4", "K7", "S2"}),
    Row("empty_streams", NO_BURSTS, {"S4"}),
    Row("cuts", None, {"L3", "L8", "L12", "L13", "S5", "S6"}),
    Row("cuts", ROUNDS, {"K3", "K6", "K8", "K9"}),
    Row("rounds_beside_pass", None, {"R6", "R7", "R8"}),
] + [Row(f"runtime_ls_{b}", ROUNDS if b == 8 else None, {f"T{b}F", f"T{b}E"}) for b in RUNTIME_LS_BS0]     # (bs0 8: the pass, unless rounds)
