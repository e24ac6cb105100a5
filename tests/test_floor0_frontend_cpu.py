"""The host front half's floor-0 records (lwf_packet_decode_ex / lwf_packet_decode_vq_ex with LWF_DECODE_FLOOR0_RECORDS):
type-0 channels come out as LWB_FLOOR_ZERO records holding exactly the amplitude and coefficient cosines the packer
encoded, everything else as without the flag, and the device's row renderer (compiled for the host) turns each record
into the front half's own dense curve, bit for bit.  No GPU needed."""
import numpy as np
import pytest

import vorbis_packer as vp
from lewton_b200 import Floor0Record
from lewton_b200 import _cabi as cabi
from lewton_b200 import frontend as fe
from test_floor0_emu import bark_cos_omega, coeff_cosines, emu, render, same_bits


@pytest.mark.parametrize("seed,channels,bs0,bs1", [(80, 2, 8, 11), (81, 1, 6, 13), (82, 3, 10, 10), (83, 6, 7, 9)])
def test_records_hold_what_was_packed_and_render_to_the_dense_curve(seed, channels, bs0, bs1):
    L = emu()
    n_rec = 0
    for k in range(20):                      # the first draw whose mappings use its type-0 floor
        if n_rec:
            break
        rng = np.random.default_rng(seed + 1000 * k)
        spec = vp.StreamSpec(rng, channels=channels, bs0=bs0, bs1=bs1, floor0=True)
        hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
        n_rec = _check_stream(L, spec, hdr)
    assert n_rec


def _check_stream(L, spec, hdr):
    n_rec = 0
    for i in range(12):
        mode = i % len(spec.modes)
        pk, info = spec.audio_packet(mode, 1, 1, p_unused=0.1)
        dense = hdr.decode_packet(pk)
        rec = hdr.decode_packet(pk, floor0_records=True)
        vq = hdr.decode_packet_vq(pk, floor0_records=True)[0] if hdr.vq_capable() else None
        want, _ = spec.expected(info)
        assert np.array_equal(dense.residue, rec.residue)
        n2 = info["n"] // 2
        for c, w in enumerate(want):
            d, r = dense.floors[c], rec.floors[c]
            if w is None or w[0] == "one":
                assert (d is None and r is None) or np.array_equal(d, r)
                continue
            fl = w[3]
            assert isinstance(r, Floor0Record) and r.amplitude == w[1]
            cosc = coeff_cosines(fl.order, w[2])
            assert np.array_equal(r.coefficients[: fl.order].view(np.uint32), cosc.view(np.uint32))
            assert not r.coefficients[fl.order:].any()
            if vq is not None:
                assert vq.floors[c].amplitude == r.amplitude and np.array_equal(vq.floors[c].coefficients, r.coefficients)
            bark = bark_cos_omega(fl.rate, fl.bark_map_size, n2)
            assert same_bits(render(L, fl, r.amplitude, cosc, bark), d), (i, c)
            n_rec += 1
    return n_rec


def test_flags_are_checked():
    rng = np.random.default_rng(84)
    spec = vp.StreamSpec(rng, channels=2, floor0=True)
    hdr = fe.Headers(spec.ident_packet(), spec.comment_packet(), spec.setup_packet())
    pk, _ = spec.audio_packet(0, 1, 1)
    dp = fe._DecodedPacket()
    kinds, ys = np.zeros(2, np.uint8), np.zeros((2, 65), np.uint32)
    res, dense = np.zeros((2, 1024), np.float32), np.zeros((2, 1024), np.float32)
    dp.floor_kind, dp.floor1_y = kinds.ctypes.data_as(cabi.u8p), ys.ctypes.data_as(cabi.u32p)
    dp.residue, dp.dense_floor = res.ctypes.data_as(cabi.fp), dense.ctypes.data_as(cabi.fp)
    assert fe.lib().lwf_packet_decode_ex(hdr._h, pk, len(pk), dp, 2) == cabi.ERR_INVALID
    dp.dense_floor = None
    assert fe.lib().lwf_packet_decode_ex(hdr._h, pk, len(pk), dp, 0) == cabi.ERR_INVALID     # dense curves need the arena
    assert fe.lib().lwf_packet_decode_ex(hdr._h, pk, len(pk), dp, fe.FLOOR0_RECORDS) == 0   # records do not
