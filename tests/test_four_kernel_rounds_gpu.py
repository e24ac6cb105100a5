"""Four-kernel batches of several rounds, queued back to back without a synchronise, against the oracle.

The four-kernel path works in rounds bounded by its IMDCT scratch.  Each round stages its descriptors in the next slot of
the staging ring and reuses the context's descriptor, spectrum and IMDCT scratch in compute-stream order only.  The
module's context is created with LWB_SCRATCH_MB=1 (262144 scratch elements), so a batch of a few 256/2048 streams takes
several rounds: its packets are cut into rounds by packet column (packet k of every chain), and with 40 channels in the
batch a long column fills 81920 elements and a short one 10240.  Each stream decodes the blocks ROUND three times: two
long and three short columns fill 194560 elements, and the next long column would overflow the scratch, so the batch
takes exactly three rounds.  Two such batches are queued behind a gate (test_queued_batches.Gate): the first uses the
ring's three slots and must return while the gate is closed, the second may wait at the ring wrap.  Each case runs first
ungated on twin streams of the same shapes, so that no arena grows behind the gate; host-memory cases make two submits
there, one per host arena set.  Every chain against the oracle: f32 PCM bit for bit, i16 PCM exactly, nothing outside the
write set of the sentinel-filled arena changed, every final stream state bit for bit, and the kernels that ran."""
import numpy as np
import pytest
import torch

import lewton_b200 as L
from helpers import ALL_KERNELS, FRONT, GENERIC, environ, launches_are_attributed
from lewton_b200 import _cabi as cabi
from test_async_batches import WIDE, AsyncCall, check_states, setups, twins
from test_queued_batches import Gate, flags

pytestmark = pytest.mark.gpu

launches_are_attributed  # (autouse)

F32P, I16I = cabi.OUT_F32_PLANAR, cabi.OUT_I16_INTERLEAVED
RESIDUE, SPECTRUM, HOST, DEVICE = cabi.ENTRY_RESIDUE, cabi.ENTRY_SPECTRUM, cabi.MEM_HOST, cabi.MEM_DEVICE
ROUND = [1, 0, 0, 0, 1]       # block flags of one round's packet columns
ROUNDS = 3
# name: (setups() key, streams per batch, LWB_FORCE_GENERIC): 40 channels either way.  10-channel streams reach the
# four-kernel path by themselves (the fused kernels and k_chain take <= 8 channels); stereo ones only when forced.
KINDS = {"wide": ("wide", 40 // WIDE, None), "stereo": ("mixed", 20, "1")}


@pytest.fixture(scope="module")
def ctx():
    with environ({"LWB_SCRATCH_MB": "1"}):      # read when the context is created
        c = L.Context(0)
    yield c
    c.close()


def queue_two(ctx, oracle, sus, gate, kind, entry, memory, fmt):
    """Two three-round batches over fresh streams of `kind`, behind the gate if one is given; then every check.  (The
    streams and page-locked arrays are freed on return, not behind a later gate: those frees wait for the device.)"""
    key, S, force = KINDS[kind]
    rng = np.random.default_rng(90)
    bf = np.tile(np.array(ROUND, np.uint8), ROUNDS)
    prev, nxt = flags(bf)
    expect = ({"k_imdct": ROUNDS, "k_overlap": ROUNDS, "k_save_state": ROUNDS}, ALL_KERNELS - GENERIC - FRONT)
    tws = twins(oracle, sus, key, S)
    calls = [AsyncCall(ctx, rng, [(tw, (bf, prev, nxt)) for tw in tws], entry, fmt, memory, expect) for _ in range(2)]
    what = (kind, entry, memory, fmt, "gated" if gate else "warm-up")
    torch.cuda.synchronize()
    if gate:
        gate.close()
    with environ({"LWB_FORCE_GENERIC": force} if force else None):
        for k, call in enumerate(calls):
            if memory == HOST:
                call.submit(ctx)
            else:
                call.decode(ctx)
            if gate and k == 0:
                if memory == HOST:
                    busy, clean = not call.ticket.done(), call.untouched()
                    if not gate.opened.query():     # both observations were made behind the closed gate
                        assert busy and clean, (what, "the batch finished behind the closed gate")
                gate.assert_closed((what, "first batch"))
    ctx.synchronize()
    for k, call in enumerate(calls):
        call.check(oracle, (what, k))
    check_states(tws, what)


@pytest.mark.parametrize("fmt", [F32P, I16I], ids=["f32_planar", "i16_interleaved"])
@pytest.mark.parametrize("memory", [DEVICE, HOST], ids=["device", "host"])
@pytest.mark.parametrize("entry", [SPECTRUM, RESIDUE], ids=["spectrum", "residue"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_three_round_batches_queued_back_to_back(ctx, oracle, kind, entry, memory, fmt):
    """Device memory through lwb_decode_chains, host memory through lwb_submit_chains from page-locked arrays."""
    sus = setups(ctx)
    gate = Gate(ctx)
    queue_two(ctx, oracle, sus, None, kind, entry, memory, fmt)
    queue_two(ctx, oracle, sus, gate, kind, entry, memory, fmt)
