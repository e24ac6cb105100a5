"""Every boundary site of the fused synthesis kernels (boundary_cases.SITES) on the GPU, against the oracle.

Each row of boundary_cases.ROWS is a case (chains that force given sites, with explicit window flags where a site needs
inconsistent ones) under a test switch.  Every batch of it, from empty streams to the batch that continues every
stream, is decoded
  * as f32 bit for bit, i16 and f16 exactly (k_long, k_long_s, k_short and k_short_g are instantiated per sample type,
    so each type is a separate copy of the boundary bodies);
  * from device memory, from host memory, and from host memory in three chunks (LWB_E2E_CHUNKS=3);
  * into an arena filled with sentinels, of which only the chains' samples may change;
  * with the exact launches per kernel that boundary_cases.Plan predicts at the device's SM count, which ties the
    model -- and so the sites it says each kernel received -- to the planner;
and the end states are held to the oracle's bit for bit.  The chain kernel alone (LWB_NO_MIXED=1) must give the same
bytes.  One residue-entry row per fused kernel runs the same boundaries behind the front stages."""
import numpy as np
import pytest
import torch

import boundary_cases as bc
import lewton_b200 as L
from helpers import (FRONT, GENERIC, RefStream, bits_equal, environ, expect_kernels, fill_guard, assert_contained,
                     launches_are_attributed, make_setup, mismatch_report)
from lewton_b200 import _cabi as cabi

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

MODES = [(0, 0), (1, 0)]             # mode 0 short, mode 1 long
FLOOR = (2, [0, 128, 12, 46, 4, 8, 16, 23, 33, 70])
FORMATS = {"f32": (cabi.OUT_F32_PLANAR, np.float32), "i16": (cabi.OUT_I16_PLANAR, np.int16),
           "f16": (cabi.OUT_F16_PLANAR, np.float16)}


@pytest.fixture(scope="module")
def ctx():
    c = L.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Reference:
    """The inputs of every batch of a case and the oracle's PCM and end state of every stream after it."""

    def __init__(self, oracle, case, residue):
        self.case, self.residue = case, residue
        C, bs0 = case.C, case.bs0
        rng = np.random.default_rng(sum(map(ord, case.name)) + 7 * residue)
        refs = [RefStream(oracle, C, bs0, 11, MODES, floors=[FLOOR] if residue else None) for _ in case.streams]
        self.batches = []
        for b in range(bc.n_batches(case)):
            coeffs, kinds, ys, wants, ends = [], [], [], [], []
            for s, st in enumerate(case.streams):
                bf, pf, nf = st[b]
                parts = []
                for i in range(len(bf)):
                    n2 = (1 << (11 if bf[i] else bs0)) // 2
                    spec = (rng.standard_normal((C, n2)) * 0.25).astype(np.float32)
                    if residue:
                        y = [[int(v) for v in rng.integers(0, 128, len(FLOOR[1]))] for _ in range(C)]
                        rc, pcm = refs[s].packet(int(bf[i]), int(pf[i]), int(nf[i]), spec, y)
                        k, yy, _ = L.DecodedPacket(int(bf[i]), spec, y).pack()
                        kinds.append(k)
                        ys.append(yy)
                    else:
                        rc, pcm = refs[s].spectrum(int(bf[i]), int(pf[i]), int(nf[i]), spec)
                    assert rc == 0, (case.name, b, s, i)
                    parts.append(pcm)
                    coeffs.append(spec.ravel())
                wants.append(np.concatenate(parts, axis=1) if parts else np.zeros((C, 0), np.float32))
                ends.append(refs[s].pwr.data().copy())
            self.batches.append((np.concatenate(coeffs), np.concatenate(kinds) if residue else None,
                                 np.concatenate(ys) if residue else None, wants, ends))
        self.oracle = oracle


_refs = {}


def reference(oracle, case, residue=False):
    key = (case.name, residue)
    if key not in _refs:
        _refs[key] = Reference(oracle, case, residue)
    return _refs[key]


def run(ctx, ref, sm, fmt, memory, env):
    """Decodes every batch of ref's case from empty streams; returns the arenas.  Checks each batch against the oracle,
    the sentinels and the launches the model predicts."""
    case = ref.case
    code, dt = FORMATS[fmt]
    su = make_setup(ctx, case.C, case.bs0, 11, modes=MODES, floors=[FLOOR])
    pwrs = [L.PreviousWindowRight(su) for _ in case.streams]
    plans = bc.plans(case, sm, env, "host" if memory == cabi.MEM_HOST else "device")
    arenas = []
    try:
        for b, (coeffs, kinds, ys, wants, ends) in enumerate(ref.batches):
            chains, ws, coff, ooff, pk = [], [], 0, 0, 0
            for s, st in enumerate(case.streams):
                bf, pf, nf = st[b]
                n = wants[s].shape[1]
                stride = ((n + 3) & ~3) + 4                       # a 4-sample gap behind every plane
                chains.append(L.ChainSpec(pwrs[s], bf, pf, nf, coeff_offset=coff, packet_index=pk, out_offset=ooff,
                                          out_stride=stride))
                ws.append((s, [(ooff + c * stride, n) for c in range(case.C) if n]))
                coff += sum(case.C * (1 << (11 if x else case.bs0)) // 2 for x in bf)
                ooff += case.C * stride
                pk += len(bf)
            pcm = fill_guard(np.zeros(ooff, dt))
            plan = plans[b]
            kw = dict(floor_kind=kinds, floor1_y=ys) if ref.residue else {}
            entry = cabi.ENTRY_RESIDUE if ref.residue else cabi.ENTRY_SPECTRUM
            with environ(env), expect_kernels(ctx, ran=dict(plan.launches), not_ran=GENERIC) as launched:
                if memory == cabi.MEM_DEVICE:
                    d_in, d_out = ctx.device_alloc(coeffs.nbytes), ctx.device_alloc(pcm.nbytes)
                    try:
                        ctx.h2d(d_in, coeffs)
                        ctx.h2d(d_out, pcm)
                        L.decode_chains(ctx, chains, entry, memory, d_in, d_out, code, **kw)
                        ctx.synchronize()
                        ctx.d2h(pcm, d_out)
                    finally:
                        ctx.device_free(d_in)
                        ctx.device_free(d_out)
                else:
                    L.decode_chains(ctx, chains, entry, memory, coeffs, pcm, code, **kw)
            assert not ref.residue or any(launched[k] for k in FRONT), launched
            what = (case.name, fmt, memory, env, b)
            assert_contained(pcm, ws, str(what))
            for s, c in enumerate(chains):
                w = wants[s]
                n = w.shape[1]
                assert (c.status, c.n_samples, c.packets_done) == (0, n, len(case.streams[s][b][0])), (what, s)
                got = np.stack([pcm[c.out_offset + k * c.out_stride:][:n] for k in range(case.C)])
                if dt == np.float32:
                    assert bits_equal(got, w), (what, s, mismatch_report(got, w))
                elif dt == np.int16:
                    assert np.array_equal(got, ref.oracle.quantise_i16(w)), (what, s)
                else:
                    assert np.array_equal(got, w.astype(np.float16)), (what, s)
                assert bits_equal(pwrs[s].data(), ends[s]), (what, s, "end state")
            arenas.append(pcm)
    finally:
        for p in pwrs:
            p.close()
    return arenas


@pytest.mark.parametrize("row", bc.ROWS, ids=lambda r: r.case + ("" if not r.env else "-" + "-".join(r.env)))
def test_site_row_matches_the_oracle(ctx, oracle, sm, row):
    """Every format and memory of a row, against the oracle, the model's launches and the chain kernel's bytes."""
    case = bc.CASES[row.case]
    reached = bc.case_sites(case, sm, row.env)
    assert row.sites <= reached, (row, sorted(row.sites - reached))
    ref = reference(oracle, case)
    f32 = run(ctx, ref, sm, "f32", cabi.MEM_DEVICE, row.env)
    run(ctx, ref, sm, "i16", cabi.MEM_HOST, row.env)
    run(ctx, ref, sm, "f16", cabi.MEM_DEVICE, row.env)
    run(ctx, ref, sm, "f16", cabi.MEM_HOST, dict(row.env or {}, **bc.CHUNKS))
    chain = run(ctx, ref, sm, "f32", cabi.MEM_HOST, dict(row.env or {}, LWB_NO_MIXED="1"))
    for a, b in zip(f32, chain):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("kernels,case,env", [("k_long_s-k_short-k_short_g", "cuts", None), ("k_long-k_short", "cuts", bc.ROUNDS)])
def test_residue_entry_rows(ctx, oracle, sm, kernels, case, env):
    """The same boundaries behind the front stages (floor 1, residue): one row per fused kernel."""
    c = bc.CASES[case]
    plans = bc.plans(c, sm, env)
    assert all(sum(p.launches[k] for p in plans) for k in kernels.split("-")), kernels
    ref = reference(oracle, c, residue=True)
    run(ctx, ref, sm, "f32", cabi.MEM_DEVICE, env)
    run(ctx, ref, sm, "i16", cabi.MEM_HOST, dict(env or {}, **bc.CHUNKS))
