"""Host-side mirror of the reference's interface for the synthesis path, over the C ABI.

Names follow lewton (src/audio.rs, src/header.rs): `PreviousWindowRight`, `read_audio_packet`,
`read_audio_packet_generic`, `get_decoded_sample_count`, `FloorTypeOne`, `Mapping`, `ModeInfo`.
The one difference is where the packet enters: the reference function takes the raw packet bytes
and entropy-decodes them first (audio.rs:921-986, host/Rust work that stays where it is); here a
packet arrives as `DecodedPacket` = what that front half produces (mode, window flags, per-channel
floor Y values, dense residue vectors).  Everything after audio.rs:988 runs on the GPU.

This module is plumbing for tests, the bench and Python callers; the product is the shared
library.  It never computes audio on the CPU: without the library / an H100 it raises.
"""
import ctypes as C
import weakref

import numpy as np

from . import _cabi as cabi


class VorbisError(Exception):
    """lib.rs:119-125"""


class AudioReadError(VorbisError):
    """audio.rs:26-41; `.kind` is the variant name, `.code` the C status."""

    def __init__(self, code, detail=""):
        self.code = code
        self.kind = {cabi.ERR_BAD_FORMAT: "AudioBadFormat", cabi.ERR_BUFFER: "BufferNotAddressable",
                     cabi.ERR_MISMATCH: "Panic", cabi.ERR_INVALID: "InvalidArgument", cabi.ERR_CUDA: "Cuda",
                     cabi.ERR_NO_DEVICE: "NoDevice"}.get(code, f"Error{code}")
        super().__init__(f"{self.kind}{': ' + detail if detail else ''}")


def _ptr(a, typ=C.c_void_p):
    return a.ctypes.data_as(typ)


class Context:
    """One per GPU (lwb_ctx)."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        rc = cabi.lib().lwb_ctx_create(device, C.byref(self._h))
        if rc:
            self._h = None
            raise AudioReadError(rc, "lwb_ctx_create failed (no sm_90 device? there is no CPU fallback)")
        self.device = device
        self._children = weakref.WeakSet()      # setups / streams: destroyed before the ctx

    def check(self, rc):
        if rc:
            raise AudioReadError(rc, cabi.lib().lwb_last_error(self._h).decode())

    def synchronize(self):
        self.check(cabi.lib().lwb_ctx_synchronize(self._h))

    @property
    def cuda_stream(self):
        return cabi.lib().lwb_ctx_cuda_stream(self._h)

    @property
    def launch_count(self):
        return cabi.lib().lwb_ctx_launch_count(self._h)

    def kernel_launches(self):
        """{kernel name: launches since creation} (lwb_ctx_kernel_launches); the counts sum to launch_count."""
        return {name: cabi.lib().lwb_ctx_kernel_launches(self._h, k) for k, name in enumerate(cabi.KERNELS)}

    def device_alloc(self, nbytes):
        p = C.c_void_p()
        self.check(cabi.lib().lwb_device_alloc(self._h, nbytes, C.byref(p)))
        return p.value

    def device_free(self, p):
        cabi.lib().lwb_device_free(self._h, p)

    def h2d(self, dst, arr):
        arr = np.ascontiguousarray(arr)
        self.check(cabi.lib().lwb_memcpy_h2d(self._h, dst, _ptr(arr), arr.nbytes))

    def d2h(self, arr, src):
        self.check(cabi.lib().lwb_memcpy_d2h(self._h, _ptr(arr), src, arr.nbytes))

    def host_alloc(self, shape, dtype):
        """A page-locked numpy array (lwb_host_alloc), as host-memory submit_chains needs; freed with its last view."""
        return np.asarray(_PinnedBlock(shape, dtype))

    def submit_chains(self, chains, entry, memory, coeffs, pcm, out_format, floor_kind=None, floor1_y=None,
                      dense_floor=None, floor_memory=cabi.MEM_HOST, vq=None):
        """lwb_submit_chains: decode_chains' arguments; queues the batch and returns its Ticket at once.  Host arrays of a
        MEM_HOST batch must be page-locked (host_alloc), and stay unchanged, and `pcm` unread, until the ticket is done."""
        chains = list(chains)
        arr, io = _marshal(chains, entry, memory, coeffs, pcm, out_format, floor_kind, floor1_y, dense_floor, floor_memory, vq)
        t = C.c_uint64()
        self.check(cabi.lib().lwb_submit_chains(self._h, arr, len(chains), C.byref(io), C.byref(t)))
        ticket = Ticket(self, t.value, (coeffs, pcm, floor_kind, floor1_y, dense_floor, vq, io), lambda: _collect(chains, arr))
        ticket.chains, ticket._arr = chains, arr
        return ticket

    def save_states(self, pwrs, buf, memory=cabi.MEM_DEVICE, offsets=None):
        """lwb_streams_save: queues copies of the states of streams `pwrs` into `buf` and returns (slots, Ticket) at once.
        Slot i (StateSlot) holds stream i's (has, len), known now, and its element offset; its [channels][len] f32 rows are
        in buf at that offset once the ticket is done.  buf: a page-locked numpy array (MEM_HOST, host_alloc) or device
        memory of this context's device (MEM_DEVICE: an integer pointer or a torch tensor).  offsets: the slots' element
        offsets, default state_offsets(pwrs) (back to back, as the states stand after every batch queued so far)."""
        pwrs = list(pwrs)
        if offsets is None:
            offsets = state_offsets(pwrs)[0]
        slots = [StateSlot(p, o) for p, o in zip(pwrs, offsets, strict=True)]
        arr = _slot_array(slots)
        t = C.c_uint64()
        self.check(cabi.lib().lwb_streams_save(self._h, arr, len(slots), memory, _addr(buf), C.byref(t)))
        for sl, a in zip(slots, arr):
            sl.len, sl.has = int(a.len), bool(a.has)
        return slots, Ticket(self, t.value, (buf, arr))

    def load_states(self, slots, buf, memory=cabi.MEM_DEVICE):
        """lwb_streams_load: queues copies of the states `slots` describe from `buf` into their streams (StateSlot.pwr, of
        this context) and returns the Ticket at once; batches queued afterwards start from them.  buf as for save_states,
        unchanged until the ticket is done.  A buffer another context saved is waited for (its save ticket) first."""
        slots = list(slots)
        arr = _slot_array(slots)
        t = C.c_uint64()
        self.check(cabi.lib().lwb_streams_load(self._h, arr, len(slots), memory, _addr(buf), C.byref(t)))
        return Ticket(self, t.value, (buf, arr))

    def close(self):
        if self._h:
            # readers (frontend.OggStreamReader) own streams and setups of their own: they go first
            for ch in [c for c in list(self._children) if not isinstance(c, (Batch, PreviousWindowRight, Setup))]:
                ch.close()
            for kind in (Batch, PreviousWindowRight, Setup):   # plans first, then streams, then setups
                for ch in [c for c in list(self._children) if isinstance(c, kind)]:
                    ch.close()
            cabi.lib().lwb_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def generate_tables(bs):
    """CachedBlocksizeDerived::from_blocksize (header_cached.rs:33-41) via the library's host code."""
    if not 6 <= bs <= 13:
        raise AudioReadError(cabi.ERR_INVALID, "blocksize out of range")
    n = 1 << bs
    a, b = np.zeros(n // 2, np.float32), np.zeros(n // 2, np.float32)
    c, w = np.zeros(n // 4, np.float32), np.zeros(n // 2, np.float32)
    br = np.zeros(n // 8, np.uint32)
    rc = cabi.lib().lwb_tables_generate(bs, _ptr(a), _ptr(b), _ptr(c), _ptr(w), _ptr(br))
    if rc:
        raise AudioReadError(rc, "blocksize out of range")
    return {"a": a, "b": b, "c": c, "window": w, "bitrev": br}


class FloorTypeOne:
    """header.rs:415-424 (fields the synthesis half reads)."""

    def __init__(self, floor1_multiplier, floor1_x_list):
        self.floor1_multiplier = int(floor1_multiplier)
        self.floor1_x_list = [int(x) for x in floor1_x_list]


class FloorTypeZero:
    """header.rs:405-412.  Without arguments its curves are computed by the host and passed dense; with the floor's
    header fields, Setup describes it to the device (Setup.set_floor0), which then also takes floor-0 records."""

    def __init__(self, order=None, rate=0, bark_map_size=0, amplitude_bits=0, amplitude_offset=0):
        self.order, self.rate, self.bark_map_size = order, int(rate), int(bark_map_size)
        self.amplitude_bits, self.amplitude_offset = int(amplitude_bits), int(amplitude_offset)


class Mapping:
    """header.rs:384-390"""

    def __init__(self, channels, magnitudes=(), angles=(), mux=None, submap_floors=(0,)):
        self.mapping_magnitudes = list(magnitudes)
        self.mapping_angles = list(angles)
        self.mapping_mux = list(mux) if mux is not None else [0] * channels
        self.mapping_submap_floors = list(submap_floors)


class ModeInfo:
    """header.rs:393-396"""

    def __init__(self, mode_blockflag, mode_mapping=0):
        self.mode_blockflag = bool(mode_blockflag)
        self.mode_mapping = int(mode_mapping)


class Setup:
    """IdentHeader (header.rs:188-211) + the SetupHeader parts (header.rs:471-477) the path reads."""

    def __init__(self, ctx, audio_channels, blocksize_0, blocksize_1, floors, mappings, modes, tables=None):
        self.ctx = ctx
        self.audio_channels, self.blocksize_0, self.blocksize_1 = audio_channels, blocksize_0, blocksize_1
        self.floors, self.mappings, self.modes = list(floors), list(mappings), list(modes)
        d = cabi.SetupDesc()
        d.audio_channels, d.blocksize_0, d.blocksize_1 = audio_channels, blocksize_0, blocksize_1
        self._keep = []
        if tables is not None:          # [(dict for bs0), (dict for bs1)] like generate_tables()
            for i, t in enumerate(tables):
                arrs = {k: np.ascontiguousarray(t[k]) for k in ("a", "b", "c", "window", "bitrev")}
                self._keep.append(arrs)
                d.tables[i].a = _ptr(arrs["a"], cabi.fp)
                d.tables[i].b = _ptr(arrs["b"], cabi.fp)
                d.tables[i].c = _ptr(arrs["c"], cabi.fp)
                d.tables[i].window = _ptr(arrs["window"], cabi.fp)
                d.tables[i].bitrev = _ptr(arrs["bitrev"], cabi.u32p)
        fl = (cabi.FloorDesc * len(self.floors))()
        for i, f in enumerate(self.floors):
            if isinstance(f, FloorTypeOne):
                fl[i].floor_type = cabi.FLOOR_TYPE_ONE
                fl[i].floor1_multiplier = f.floor1_multiplier
                fl[i].floor1_values = len(f.floor1_x_list)
                for k, x in enumerate(f.floor1_x_list[: cabi.MAX_POSTS]):
                    fl[i].floor1_x_list[k] = x
            else:
                fl[i].floor_type = cabi.FLOOR_TYPE_ZERO
        mp = (cabi.MappingDesc * len(self.mappings))()
        for i, m in enumerate(self.mappings):
            mp[i].coupling_steps = len(m.mapping_magnitudes)
            mp[i].submaps = len(m.mapping_submap_floors)
            for k, (a, b) in enumerate(zip(m.mapping_magnitudes, m.mapping_angles)):
                mp[i].magnitudes[k], mp[i].angles[k] = a, b
            for k, v in enumerate(m.mapping_mux):
                mp[i].mux[k] = v
            for k, v in enumerate(m.mapping_submap_floors):
                mp[i].submap_floors[k] = v
        md = (cabi.ModeDesc * len(self.modes))()
        for i, m in enumerate(self.modes):
            md[i].blockflag, md[i].mapping = int(m.mode_blockflag), m.mode_mapping
        d.n_floors, d.floors = len(self.floors), fl
        d.n_mappings, d.mappings = len(self.mappings), mp
        d.n_modes, d.modes = len(self.modes), md
        self._h = C.c_void_p()
        rc = cabi.lib().lwb_setup_create(ctx._h, C.byref(d), C.byref(self._h))
        if rc:
            self._h = None
            raise AudioReadError(rc, cabi.lib().lwb_last_error(ctx._h).decode())
        ctx._children.add(self)
        for i, f in enumerate(self.floors):
            if isinstance(f, FloorTypeZero) and f.order is not None:
                self.set_floor0(i, f.order, f.rate, f.bark_map_size, f.amplitude_bits, f.amplitude_offset)

    def set_floor0(self, floor_index, order, rate, bark_map_size, amplitude_bits, amplitude_offset, bark_cos_omega=(None, None)):
        """lwb_setup_set_floor0: describe type-0 floor `floor_index` so that packets may carry it as a floor-0 record
        (DecodedPacket floors given as Floor0Record); bark_cos_omega: the two cached tables (n/2 float32 each) or None
        to generate them."""
        d = cabi.Floor0Desc()
        d.order, d.amplitude_bits, d.amplitude_offset = order, amplitude_bits, amplitude_offset
        d.rate, d.bark_map_size = rate, bark_map_size
        keep = []
        for i, t in enumerate(bark_cos_omega):
            if t is not None:
                keep.append(np.ascontiguousarray(t, np.float32))
                d.bark_cos_omega[i] = _ptr(keep[-1], cabi.fp)
        self.ctx.check(cabi.lib().lwb_setup_set_floor0(self._h, floor_index, C.byref(d)))

    def set_output_mix(self, matrix):
        """lwb_setup_set_output_mix: chains of this setup's streams write K = len(matrix) output channels, output k the
        f32 sum over input channels c (ascending, zero coefficients skipped) of matrix[k][c] * sample_c; None clears the
        mix.  matrix: [K][audio_channels], 1 <= K <= 8 (mix_mono, mix_select, mix_wav_order build the common ones).  Only
        before the setup's first stream is opened."""
        if matrix is None:
            self.ctx.check(cabi.lib().lwb_setup_set_output_mix(self._h, 0, None))
            return
        m = np.ascontiguousarray(matrix, np.float32)
        if m.ndim != 2 or m.shape[1] != self.audio_channels:
            raise ValueError(f"matrix: [K][{self.audio_channels}] expected, got shape {m.shape}")
        self.ctx.check(cabi.lib().lwb_setup_set_output_mix(self._h, m.shape[0], _ptr(m, cabi.fp)))

    @property
    def output_channels(self):
        """K: the channels a chain of this setup writes (lwb_setup_output_channels); audio_channels without a mix."""
        return cabi.lib().lwb_setup_output_channels(self._h)

    @classmethod
    def _adopt(cls, ctx, handle, audio_channels, blocksize_0, blocksize_1, mode_blockflags=()):
        """Wrap an lwb_setup built by the library itself (lwf_headers_make_setup)."""
        self = cls.__new__(cls)
        self.ctx = ctx
        self.audio_channels, self.blocksize_0, self.blocksize_1 = audio_channels, blocksize_0, blocksize_1
        self.floors, self.mappings = [], []
        self.modes = [ModeInfo(bool(b)) for b in mode_blockflags]
        self._keep = []
        self._h = C.c_void_p(handle)
        ctx._children.add(self)
        return self

    def blocksize(self, mode_number):
        if not 0 <= mode_number < len(self.modes):
            raise AudioReadError(cabi.ERR_BAD_FORMAT, "mode number out of range (audio.rs:926-930)")
        return 1 << (self.blocksize_1 if self.modes[mode_number].mode_blockflag else self.blocksize_0)

    def close(self):
        if self._h:
            if self.ctx._h:
                cabi.lib().lwb_setup_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


NO_LIMIT = (1 << 64) - 1      # lwb_stream_set_window: a window without an end


class PreviousWindowRight:
    """audio.rs:847-861 -- the only inter-packet state, resident on the device (lwb_stream)."""

    def __init__(self, setup, _handle=None):
        self.setup = setup
        self._h = _handle or C.c_void_p()
        if _handle is None:
            setup.ctx.check(cabi.lib().lwb_stream_open(setup.ctx._h, setup._h, C.byref(self._h)))
        setup.ctx._children.add(self)

    @classmethod
    def new(cls, setup):
        return cls(setup)

    def is_empty(self):
        return bool(cabi.lib().lwb_stream_is_empty(self._h))

    def reset(self):
        cabi.lib().lwb_stream_reset(self._h)

    def clone(self):
        h = C.c_void_p()
        self.setup.ctx.check(cabi.lib().lwb_stream_clone(self._h, C.byref(h)))
        return PreviousWindowRight(self.setup, h)

    def set_window(self, skip=0, limit=None):
        """Output window (lwb_stream_set_window): of the samples the next packets produce, drop the first `skip` per
        channel, write the next `limit` (None: no end) and none after them.  The state advances as without a window;
        reset() leaves the window alone, so a seek is reset() then set_window(skip).  Batches report the samples
        written."""
        limit = NO_LIMIT if limit is None else int(limit)
        if skip < 0 or not 0 <= limit <= NO_LIMIT:
            raise ValueError("skip and limit must be >= 0 (limit None: no end)")
        self.setup.ctx.check(cabi.lib().lwb_stream_set_window(self._h, int(skip), limit))

    @property
    def window(self):
        """What is left of the window: (skip still to drop, limit still to write or None for no end)."""
        skip, limit = C.c_uint64(), C.c_uint64()
        self.setup.ctx.check(cabi.lib().lwb_stream_window(self._h, C.byref(skip), C.byref(limit)))
        return skip.value, None if limit.value == NO_LIMIT else limit.value

    def __len__(self):
        return cabi.lib().lwb_stream_state_len(self._h)

    def data(self):
        if self.is_empty():
            return None
        out = np.zeros((self.setup.audio_channels, len(self)), np.float32)
        self.setup.ctx.check(cabi.lib().lwb_stream_export_state(self._h, _ptr(out)))
        return out

    def set_data(self, arr):
        arr = np.ascontiguousarray(arr, np.float32)
        assert arr.shape[0] == self.setup.audio_channels
        self.setup.ctx.check(cabi.lib().lwb_stream_import_state(self._h, _ptr(arr), arr.shape[1]))

    def close(self):
        if self._h:
            if self.setup.ctx._h:
                cabi.lib().lwb_stream_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class StateSlot:
    """One stream's state in a state buffer (lwb_state_slot): [channels][len] f32 rows at element `offset`; has False is
    the empty state of PreviousWindowRight::new().  Context.save_states fills len and has; Context.load_states reads them
    into `pwr`."""

    def __init__(self, pwr, offset, len=0, has=False):
        self.pwr, self.offset, self.len, self.has = pwr, int(offset), int(len), bool(has)

    def __repr__(self):
        return f"StateSlot(offset={self.offset}, len={self.len}, has={self.has})"


def state_offsets(pwrs, lengths=None):
    """Element offsets that lay the states of streams `pwrs` out back to back in one state buffer, each starting at a
    multiple of 4 floats (so the copies move float4s), and the buffer's size in elements: (offsets, total).
    lengths: the state length of each stream; by default its len() now, which is what a save queued now writes.  Pass
    blocksize_1 // 2 of each stream's setup for a layout that holds any state the streams may have later."""
    pwrs = list(pwrs)
    lengths = [len(p) for p in pwrs] if lengths is None else [int(n) for n in lengths]
    offsets, total = [], 0
    for p, n in zip(pwrs, lengths, strict=True):
        offsets.append(total)
        total += (p.setup.audio_channels * n + 3) // 4 * 4
    return offsets, total


def _slot_array(slots):
    arr = (cabi.StateSlot * len(slots))()
    for a, sl in zip(arr, slots):
        a.stream, a.offset, a.len, a.has = sl.pwr._h, sl.offset, sl.len, int(sl.has)
    return arr


def _addr(x):
    """The address of an arena: a numpy array's data, a torch tensor's data_ptr(), or an integer pointer (None: NULL)."""
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    return int(x)


class Floor0Record:
    """DecodedFloor::TypeZero as floor_zero_decode returns it (audio.rs:109-158): the amplitude and the coefficient
    cosines; packed as the LWB_FLOOR_ZERO record of a floor1_y row."""

    def __init__(self, amplitude, coefficients):
        self.amplitude = int(amplitude)
        self.coefficients = np.ascontiguousarray(coefficients, np.float32)
        if not 2 <= len(self.coefficients) <= cabi.MAX_POSTS - 2:
            raise ValueError("a floor-0 record holds 2..63 coefficients")

    def words(self):
        w = np.zeros(cabi.MAX_POSTS, np.uint32)
        w[0], w[1] = self.amplitude & 0xFFFFFFFF, self.amplitude >> 32
        w[2: 2 + len(self.coefficients)] = self.coefficients.view(np.uint32)
        return w


class DecodedPacket:
    """What audio.rs:921-986 hands to the synthesis half.

    floors: per channel  None (DecodedFloor::Unused) | sequence of floor1 Y values
            (DecodedFloor::TypeOne) | float32 ndarray of n/2 (a floor-0 curve computed by the host) |
            Floor0Record (DecodedFloor::TypeZero: the device computes the curve)
    residue: [channels][n/2] float32
    """

    def __init__(self, mode_number, residue, floors, prev_window_flag=True, next_window_flag=True):
        self.mode_number = mode_number
        self.prev_window_flag, self.next_window_flag = bool(prev_window_flag), bool(next_window_flag)
        self.residue = np.ascontiguousarray(residue, np.float32)
        self.floors = list(floors)

    def pack(self):
        ch, n2 = self.residue.shape
        kinds = np.zeros(ch, np.uint8)
        ys = np.zeros((ch, cabi.MAX_POSTS), np.uint32)
        dense = None
        for c, f in enumerate(self.floors):
            if f is None:
                kinds[c] = cabi.FLOOR_UNUSED
            elif isinstance(f, Floor0Record):
                kinds[c] = cabi.FLOOR_ZERO
                ys[c] = f.words()
            elif isinstance(f, np.ndarray) and f.dtype.kind == "f":
                kinds[c] = cabi.FLOOR_DENSE
                if dense is None:
                    dense = np.zeros((ch, n2), np.float32)
                dense[c] = f
            else:
                kinds[c] = cabi.FLOOR_ONE
                ys[c, : len(f)] = np.asarray(f, np.uint32)
        return kinds, ys, dense


# (sample, interleaved) -> (LWB_OUT_*, numpy dtype).  "f16": IEEE binary16, the f32 sample rounded to nearest even.
# "i32" / "i24": the f32 sample times 2^31 / 2^23, truncated toward zero and saturated (NaN -> 0); an i24 element is 3
# bytes, little-endian two's complement, so its dtype is the 3-byte void type I24 (widen with i24_to_i32).
I24 = np.dtype("V3")
_FORMATS = {("f32", False): (cabi.OUT_F32_PLANAR, np.float32), ("i16", False): (cabi.OUT_I16_PLANAR, np.int16),
            ("f32", True): (cabi.OUT_F32_INTERLEAVED, np.float32), ("i16", True): (cabi.OUT_I16_INTERLEAVED, np.int16),
            ("f16", False): (cabi.OUT_F16_PLANAR, np.float16), ("f16", True): (cabi.OUT_F16_INTERLEAVED, np.float16),
            ("i32", False): (cabi.OUT_I32_PLANAR, np.int32), ("i32", True): (cabi.OUT_I32_INTERLEAVED, np.int32),
            ("i24", False): (cabi.OUT_I24_PLANAR, I24), ("i24", True): (cabi.OUT_I24_INTERLEAVED, I24)}


def sample_format(sample, interleaved=False):
    """(LWB_OUT_* format, numpy dtype) of sample type "f32" | "i16" | "f16" | "i32" | "i24" in the planar or interleaved
    layout (KeyError for any other sample type)."""
    return _FORMATS[(sample, bool(interleaved))]


def i24_to_i32(arr):
    """I24 PCM widened to int32, sign-extended.  arr: a numpy array of I24 elements (any shape), or a numpy array or torch
    tensor of uint8 whose last dimension holds 3 bytes per sample (a torch tensor stays on its device)."""
    if hasattr(arr, "data_ptr"):                                         # torch
        import torch
        if arr.dtype != torch.uint8 or arr.shape[-1] % 3:
            raise ValueError("i24_to_i32: a torch tensor must be uint8 with 3 bytes per sample in its last dimension")
        b = arr.reshape(*arr.shape[:-1], arr.shape[-1] // 3, 3).to(torch.int32)
        v = b[..., 0] | (b[..., 1] << 8) | (b[..., 2] << 16)
        return (v << 8) >> 8
    a = np.ascontiguousarray(arr)
    if a.dtype == I24:
        b = a.view(np.uint8).reshape(a.shape + (3,))
    elif a.dtype == np.uint8 and a.ndim and a.shape[-1] % 3 == 0:
        b = a.reshape(a.shape[:-1] + (a.shape[-1] // 3, 3))
    else:
        raise ValueError("i24_to_i32: need I24 elements or uint8 bytes, 3 per sample in the last dimension")
    v = b[..., 0].astype(np.uint32) | (b[..., 1].astype(np.uint32) << 8) | (b[..., 2].astype(np.uint32) << 16)
    return (v << 8).view(np.int32) >> 8


def mix_mono(channels):
    """The output mix (Setup.set_output_mix) of a mono downmix: one row of weights 1/channels (f32)."""
    return np.full((1, channels), np.float32(1) / np.float32(channels), np.float32)


def mix_select(channels, outputs):
    """The output mix that writes input channels `outputs` (indices, in Vorbis order; repeats duplicate a channel) as the
    output channels, in that order: bit-exact copies."""
    m = np.zeros((len(outputs), channels), np.float32)
    for k, c in enumerate(outputs):
        if not 0 <= c < channels:
            raise ValueError(f"channel {c} out of range for {channels} channels")
        m[k, c] = 1
    return m


# Vorbis I section 4.3.9 channel order -> the WAVEFORMATEXTENSIBLE channel-mask order (FL FR FC LFE BL BR FLC FRC BC SL SR)
# that WAV files, ALSA and most PCM pipelines use: entry k is the Vorbis channel that becomes output channel k.
_WAV_ORDER = {1: (0,), 2: (0, 1),
              3: (0, 2, 1),                     # L C R -> L R C
              4: (0, 1, 2, 3),                  # FL FR RL RR (already in mask order)
              5: (0, 2, 1, 3, 4),               # FL C FR RL RR -> FL FR FC BL BR
              6: (0, 2, 1, 5, 3, 4),            # FL C FR RL RR LFE -> FL FR FC LFE BL BR
              7: (0, 2, 1, 6, 5, 3, 4),         # FL C FR SL SR RC LFE -> FL FR FC LFE BC SL SR
              8: (0, 2, 1, 7, 5, 6, 3, 4)}      # FL C FR SL SR RL RR LFE -> FL FR FC LFE BL BR SL SR


def mix_wav_order(channels):
    """The output mix that reorders 1 to 8 channels from Vorbis order to WAV order (a permutation: bit-exact)."""
    if channels not in _WAV_ORDER:
        raise ValueError("WAV order is defined for 1 to 8 channels")
    return mix_select(channels, _WAV_ORDER[channels])


def get_decoded_sample_count(setup, mode_number, prev_window_flag=True, next_window_flag=True):
    """audio.rs:874-909 for an already parsed packet header."""
    n = C.c_uint32()
    rc = cabi.lib().lwb_decoded_sample_count(setup._h, mode_number, int(prev_window_flag), int(next_window_flag),
                                             C.byref(n))
    if rc:
        raise AudioReadError(rc)
    return n.value


def read_audio_packet_generic(setup, packet, pwr, sample="f32", interleaved=False):
    """audio.rs:919-1160 (back half).  Returns planar [channels][len] (Vec<Vec<S>>) or
    interleaved [len][channels] (InterleavedSamples<S>), channels = setup.output_channels; len == 0 for the first packet
    after a reset.
    Raises AudioReadError (kind 'AudioBadFormat' for the guard at audio.rs:1107-1111)."""
    fmt, dt = sample_format(sample, interleaved)
    ch = setup.output_channels
    cap = setup.blocksize(packet.mode_number)
    kinds, ys, dense = packet.pack()
    p = cabi.Packet()
    p.mode_number = packet.mode_number
    p.prev_window_flag, p.next_window_flag = int(packet.prev_window_flag), int(packet.next_window_flag)
    p.floor_kind = _ptr(kinds, cabi.u8p)
    p.floor1_y = _ptr(ys, cabi.u32p)
    if dense is not None:
        p.dense_floor = _ptr(dense, cabi.fp)
    p.residue = _ptr(packet.residue, cabi.fp)
    out = np.zeros((cap, ch) if interleaved else (ch, cap), dt)
    n = C.c_size_t()
    rc = cabi.lib().lwb_decode_packet(pwr._h, C.byref(p), fmt, _ptr(out), cap, C.byref(n))
    if rc:
        raise AudioReadError(rc, cabi.lib().lwb_last_error(setup.ctx._h).decode())
    return out[: n.value].copy() if interleaved else out[:, : n.value].copy()


def read_audio_packet(setup, packet, pwr):
    """audio.rs:1170-1173: Vec<Vec<i16>>."""
    return read_audio_packet_generic(setup, packet, pwr, sample="i16", interleaved=False)


def decode_spectrum(setup, mode_number, spectrum, pwr, prev_window_flag=True, next_window_flag=True, sample="f32",
                    interleaved=False):
    """Entry at the record_pre_mdct tap (audio.rs:1041): spectrum [channels][n/2] = floor x residue."""
    fmt, dt = sample_format(sample, interleaved)
    ch = setup.output_channels
    cap = setup.blocksize(mode_number)
    sp = np.ascontiguousarray(spectrum, np.float32)
    out = np.zeros((cap, ch) if interleaved else (ch, cap), dt)
    n = C.c_size_t()
    rc = cabi.lib().lwb_decode_spectrum(pwr._h, mode_number, int(prev_window_flag), int(next_window_flag), _ptr(sp), fmt,
                                        _ptr(out), cap, C.byref(n))
    if rc:
        raise AudioReadError(rc, cabi.lib().lwb_last_error(setup.ctx._h).decode())
    return out[: n.value].copy() if interleaved else out[:, : n.value].copy()


def debug_taps(setup, packet, pwr):
    """The reference's record_* taps (lib.rs:56-94): post-inverse-coupling residue, pre-MDCT
    spectrum, post-MDCT samples.  Does not modify the state."""
    ch = setup.audio_channels
    n = setup.blocksize(packet.mode_number)
    kinds, ys, dense = packet.pack()
    p = cabi.Packet()
    p.mode_number = packet.mode_number
    p.prev_window_flag, p.next_window_flag = int(packet.prev_window_flag), int(packet.next_window_flag)
    p.floor_kind, p.floor1_y = _ptr(kinds, cabi.u8p), _ptr(ys, cabi.u32p)
    if dense is not None:
        p.dense_floor = _ptr(dense, cabi.fp)
    p.residue = _ptr(packet.residue, cabi.fp)
    a, b, c = (np.zeros((ch, n // 2), np.float32), np.zeros((ch, n // 2), np.float32), np.zeros((ch, n), np.float32))
    setup.ctx.check(cabi.lib().lwb_debug_packet_taps(pwr._h, C.byref(p), _ptr(a), _ptr(b), _ptr(c)))
    return a, b, c


class ChainSpec:
    """One stream's run of consecutive packets inside a batch (lwb_chain)."""

    def __init__(self, pwr, mode_numbers, prev_flags=None, next_flags=None, coeff_offset=0, packet_index=0,
                 out_offset=0, out_stride=0):
        self.pwr = pwr
        self.modes = np.ascontiguousarray(mode_numbers, np.uint8)
        self.prev = None if prev_flags is None else np.ascontiguousarray(prev_flags, np.uint8)
        self.next = None if next_flags is None else np.ascontiguousarray(next_flags, np.uint8)
        self.coeff_offset, self.packet_index = coeff_offset, packet_index
        self.out_offset, self.out_stride = out_offset, out_stride
        self.n_samples = self.packets_done = self.status = 0


class Batch:
    """A prepared lwb_decode_chains call: the lwb_chain array and lwb_batch_io are built once, so a
    hot loop pays only the C call (the per-step Python cost of marshalling thousands of chains
    would otherwise exceed the kernel time)."""

    def __init__(self, ctx, chains, entry, memory, coeffs, pcm, out_format, floor_kind=None, floor1_y=None,
                 dense_floor=None, floor_memory=cabi.MEM_HOST, vq=None):
        """vq: LWB_ENTRY_VQ arrays (runs, run_offsets, entries, entry_offsets): numpy arrays or device pointers."""
        self.ctx, self.chains = ctx, list(chains)
        self._keep = (coeffs, pcm, floor_kind, floor1_y, dense_floor, vq)
        self._arr, self._io = _marshal(self.chains, entry, memory, coeffs, pcm, out_format, floor_kind, floor1_y,
                                       dense_floor, floor_memory, vq)
        self._n = len(self.chains)
        self._plan = C.c_void_p()
        ctx.check(cabi.lib().lwb_plan_create(ctx._h, self._arr, self._n, C.byref(self._io), C.byref(self._plan)))
        ctx._children.add(self)
        self._fn = cabi.lib().lwb_plan_execute

    def run(self):
        """One submission (lwb_plan_execute).  Results land in the chain array; collect() copies them back."""
        rc = self._fn(self._plan)
        if rc:
            self.ctx.check(rc)

    def close(self):
        if self._plan:
            if self.ctx._h:
                cabi.lib().lwb_plan_destroy(self._plan)
            self._plan = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def collect(self):
        return _collect(self.chains, self._arr)


class _PinnedBlock:
    """Owner of one lwb_host_alloc block, exposed to numpy as an array; freed when the last array over it goes."""

    def __init__(self, shape, dtype):
        dtype = np.dtype(dtype)
        shape = (int(shape),) if np.isscalar(shape) else tuple(int(s) for s in shape)
        nbytes = int(np.prod(shape, dtype=np.int64)) * dtype.itemsize
        self._p = cabi.lib().lwb_host_alloc(nbytes)
        if not self._p:
            raise AudioReadError(cabi.ERR_CUDA, f"lwb_host_alloc({nbytes}) failed")
        self.__array_interface__ = {"data": (self._p, False), "shape": shape, "typestr": dtype.str, "descr": dtype.descr,
                                    "version": 3}

    def __del__(self):
        if getattr(self, "_p", None):
            cabi.lib().lwb_host_free(self._p)
            self._p = None


class Ticket:
    """Work queued on a context: a batch (Context.submit_chains, StreamBatcher.submit, OggStreamReaders.read) or a copy
    of stream states (save_states, load_states).  It keeps every array the work reads or writes (`keep`) alive until it
    is done; wait() returns result(), built from the results the library wrote before the queuing call returned."""

    def __init__(self, ctx, ticket, keep, result=list):
        self.ctx, self.id, self._keep, self._result = ctx, ticket, keep, result

    def done(self):
        """lwb_ticket_query: whether every copy and kernel of the work has finished.  Never blocks."""
        if self._keep is not None:
            d = C.c_int()
            self.ctx.check(cabi.lib().lwb_ticket_query(self.ctx._h, self.id, C.byref(d)))
            if not d.value:
                return False
            self._keep = None
        return True

    def wait(self):
        """lwb_ticket_wait; returns the results: submit_chains' chains with theirs, StreamBatcher.submit's
        [(n_samples, packets_done, status)], OggStreamReaders.read's [ReadResult], none for save_states and load_states."""
        if self._keep is not None:
            self.ctx.check(cabi.lib().lwb_ticket_wait(self.ctx._h, self.id))
            self._keep = None
        return self._result()


def _marshal(chains, entry, memory, coeffs, pcm, out_format, floor_kind, floor1_y, dense_floor, floor_memory, vq):
    """The lwb_chain array and lwb_batch_io of a batch (they point into the ChainSpecs' arrays and the arenas)."""
    arr = (cabi.Chain * len(chains))()
    for i, c in enumerate(chains):
        arr[i].stream = c.pwr._h
        arr[i].n_packets = len(c.modes)
        arr[i].mode_numbers = _ptr(c.modes, cabi.u8p)
        if c.prev is not None:
            arr[i].prev_window_flags = _ptr(c.prev, cabi.u8p)
        if c.next is not None:
            arr[i].next_window_flags = _ptr(c.next, cabi.u8p)
        arr[i].coeff_offset, arr[i].packet_index = c.coeff_offset, c.packet_index
        arr[i].out_offset, arr[i].out_stride = c.out_offset, c.out_stride

    addr = _addr
    io = cabi.BatchIo()
    io.entry, io.memory, io.out_format = entry, memory, out_format
    io.coeffs, io.pcm, io.dense_floor = addr(coeffs), addr(pcm), addr(dense_floor)
    io.floor_kind, io.floor1_y = addr(floor_kind), addr(floor1_y)
    io.floor_memory = floor_memory
    if vq is not None:
        io.vq_runs, io.vq_run_offsets, io.vq_entries, io.vq_entry_offsets = (addr(x) for x in vq)
    return arr, io


def _collect(chains, arr):
    for i, c in enumerate(chains):
        c.n_samples, c.packets_done, c.status = arr[i].n_samples, arr[i].packets_done, arr[i].status
    return chains


def decode_chains(ctx, chains, entry, memory, coeffs, pcm, out_format, floor_kind=None, floor1_y=None,
                  dense_floor=None, floor_memory=cabi.MEM_HOST, vq=None):
    """lwb_decode_chains.  coeffs/pcm/dense_floor: numpy arrays (MEM_HOST) or integer device
    pointers (MEM_DEVICE); floor_kind/floor1_y: numpy arrays (floor_memory MEM_HOST) or integer
    device pointers (MEM_DEVICE).  A MEM_DEVICE batch returns once its work is queued on ctx.cuda_stream."""
    chains = list(chains)
    arr, io = _marshal(chains, entry, memory, coeffs, pcm, out_format, floor_kind, floor1_y, dense_floor, floor_memory, vq)
    ctx.check(cabi.lib().lwb_decode_chains(ctx._h, arr, len(chains), C.byref(io)))
    return _collect(chains, arr)
