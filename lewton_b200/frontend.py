"""Host front half (include/lewton_frontend.h) -- ctypes mirror of the reference's public reading API:

  read_headers / Headers          header.rs:221, :309, :1082  (IdentHeader, CommentHeader, SetupHeader)
  Headers.decode_packet           audio.rs:919-986            (front half of read_audio_packet_generic)
  Headers.decoded_sample_count    audio.rs:874-909            (get_decoded_sample_count)
  OggPacketReader                 ogg::PacketReader as inside_ogg.rs uses it
  OggStreamReader                 inside_ogg.rs:60-227        (read_dec_packet, read_dec_packet_itl, read_dec_packet_generic,
                                                              get_last_absgp)
  OggStreamReaders                many OggStreamReaders advanced, sought and skipped by batched calls (lwf_readers)

The entropy decode is CPU work by nature and runs on the host; synthesis goes through the CUDA back
half (lwb_decode_packet / lwb_decode_chains)."""
import ctypes as C

import numpy as np

from . import _cabi as cabi
from .api import AudioReadError, DecodedPacket, Floor0Record, Setup, Ticket, sample_format

(ERR_END_OF_PACKET, ERR_NOT_VORBIS_HEADER, ERR_UNSUPPORTED_VERSION, ERR_HEADER_BAD_FORMAT, ERR_HEADER_BAD_TYPE,
 ERR_HEADER_IS_AUDIO, ERR_UTF8, ERR_AUDIO_IS_HEADER, ERR_OGG, ERR_NO_MORE_PACKETS) = range(16, 26)

SYMBOLS = ["lwf_headers_parse", "lwf_headers_destroy", "lwf_headers_info", "lwf_headers_comment", "lwf_headers_make_setup",
           "lwf_headers_make_setup_floor0", "lwf_packet_decode", "lwf_packet_decode_ex", "lwf_packet_decode_vq", "lwf_packet_decode_vq_ex", "lwf_headers_vq_capable", "lwf_decoded_sample_count", "lwf_ogg_open", "lwf_ogg_close", "lwf_ogg_next_packet",
           "lwf_reader_open", "lwf_reader_close", "lwf_reader_headers", "lwf_reader_read_dec_packet", "lwf_reader_last_absgp",
           "lwf_reader_skip_samples_linear", "lwf_reader_seek_absgp_pg",
           "lwf_batcher_create", "lwf_batcher_destroy", "lwf_batcher_set_entry", "lwf_batcher_decode", "lwf_batcher_last_timing",
           "lwf_batcher_last_input_bytes", "lwf_batcher_set_floor0", "lwf_batcher_submit", "lwf_batcher_add_headers",
           "lwf_readers_create", "lwf_readers_destroy", "lwf_readers_add", "lwf_readers_headers", "lwf_readers_last_absgp",
           "lwf_readers_setup_count", "lwf_readers_last_timing", "lwf_readers_read",
           "lwf_debug_float32_unpack", "lwf_debug_lookup1_values", "lwf_debug_ilog", "lwf_debug_read_bits", "lwf_debug_huffman",
           "lwf_debug_decode_loop"]


VQ_RUN_DTYPE = np.dtype([("pos", np.uint16), ("first", np.uint16), ("book", np.uint8), ("pass_kind", np.uint8), ("aux", np.uint8),
                         ("count", np.uint8)])                                              # lwb_vq_run


class HeaderReadError(Exception):
    """header.rs:35-44"""

    def __init__(self, code):
        names = {ERR_END_OF_PACKET: "EndOfPacket", ERR_NOT_VORBIS_HEADER: "NotVorbisHeader",
                 ERR_UNSUPPORTED_VERSION: "UnsupportedVorbisVersion", ERR_HEADER_BAD_FORMAT: "HeaderBadFormat",
                 ERR_HEADER_BAD_TYPE: "HeaderBadType", ERR_HEADER_IS_AUDIO: "HeaderIsAudio", ERR_UTF8: "Utf8DecodeError",
                 cabi.ERR_BUFFER: "BufferNotAddressable"}
        super().__init__(names.get(code, "code %d" % code))
        self.code = code


class OggReadError(Exception):
    pass


class Info(C.Structure):
    _fields_ = [("audio_channels", C.c_uint8), ("blocksize_0", C.c_uint8), ("blocksize_1", C.c_uint8),
                ("audio_sample_rate", C.c_uint32), ("bitrate_maximum", C.c_int32), ("bitrate_nominal", C.c_int32),
                ("bitrate_minimum", C.c_int32), ("n_codebooks", C.c_uint32), ("n_floors", C.c_uint32),
                ("n_residues", C.c_uint32), ("n_mappings", C.c_uint32), ("n_modes", C.c_uint32), ("n_comments", C.c_uint32)]


class _DecodedPacket(C.Structure):
    _fields_ = [("mode_number", C.c_uint8), ("blockflag", C.c_uint8), ("prev_window_flag", C.c_uint8),
                ("next_window_flag", C.c_uint8), ("n", C.c_uint32), ("floor_kind", cabi.u8p), ("floor1_y", cabi.u32p),
                ("dense_floor", cabi.fp), ("residue", cabi.fp)]


class _OggPacket(C.Structure):
    _fields_ = [("data", cabi.u8p), ("len", C.c_size_t), ("stream_serial", C.c_uint32), ("absgp_page", C.c_uint64),
                ("first_in_stream", C.c_uint8), ("last_in_stream", C.c_uint8), ("first_in_page", C.c_uint8),
                ("last_in_page", C.c_uint8)]


class _StreamJob(C.Structure):
    _fields_ = [("stream", C.c_void_p), ("n_packets", C.c_uint32), ("packets", C.POINTER(C.c_char_p)),
                ("lengths", C.POINTER(C.c_size_t)), ("out_offset", C.c_uint64), ("out_stride", C.c_uint64),
                ("n_samples", C.c_uint32), ("packets_done", C.c_uint32), ("status", C.c_int32)]


class _ReadJob(C.Structure):
    _fields_ = [("reader", C.c_uint32), ("max_packets", C.c_uint32), ("out_offset", C.c_uint64), ("out_stride", C.c_uint64),
                ("packet_samples", cabi.u32p), ("n_packets", C.c_uint32), ("n_samples", C.c_uint32), ("channels", C.c_uint8),
                ("next_chained", C.c_uint8), ("ended", C.c_uint8), ("reserved", C.c_uint8), ("status", C.c_int32)]


class _SkipJob(C.Structure):
    _fields_ = [("reader", C.c_uint32), ("out_channels", C.c_uint32), ("to_skip", C.c_uint64), ("out_offset", C.c_uint64),
                ("out_stride", C.c_uint64), ("left_to_skip", C.c_uint64), ("n_samples", C.c_uint32), ("got_packet", C.c_uint8),
                ("channels", C.c_uint8), ("reserved", C.c_uint8 * 2), ("status", C.c_int32)]


_declared = False


def lib():
    global _declared
    L = cabi.lib()
    if not _declared:
        vp, sz = C.c_void_p, C.c_size_t
        L.lwf_headers_parse.argtypes = [C.c_char_p, sz, C.c_char_p, sz, C.c_char_p, sz, C.POINTER(vp)]
        L.lwf_headers_destroy.argtypes = [vp]
        L.lwf_headers_destroy.restype = None
        L.lwf_headers_info.argtypes = [vp, C.POINTER(Info)]
        L.lwf_headers_comment.argtypes = [vp, C.c_int, C.c_char_p, sz]
        L.lwf_headers_comment.restype = sz
        L.lwf_headers_make_setup.argtypes = [vp, vp, C.POINTER(vp)]
        L.lwf_packet_decode.argtypes = [vp, C.c_char_p, sz, C.POINTER(_DecodedPacket)]
        L.lwf_packet_decode_ex.argtypes = [vp, C.c_char_p, sz, C.POINTER(_DecodedPacket), C.c_int]
        L.lwf_headers_make_setup_floor0.argtypes = [vp, vp, C.POINTER(vp)]
        L.lwf_batcher_set_floor0.argtypes = [vp, C.c_int]
        L.lwf_batcher_last_input_bytes.argtypes = [vp]
        L.lwf_batcher_last_input_bytes.restype = C.c_uint64
        L.lwf_decoded_sample_count.argtypes = [vp, C.c_char_p, sz, C.POINTER(sz)]
        L.lwf_ogg_open.argtypes = [C.c_char_p, sz, C.POINTER(vp)]
        L.lwf_ogg_close.argtypes = [vp]
        L.lwf_ogg_close.restype = None
        L.lwf_ogg_next_packet.argtypes = [vp, C.POINTER(_OggPacket)]
        L.lwf_reader_open.argtypes = [vp, C.c_char_p, sz, C.POINTER(vp)]
        L.lwf_reader_close.argtypes = [vp]
        L.lwf_reader_close.restype = None
        L.lwf_reader_headers.argtypes = [vp]
        L.lwf_reader_headers.restype = vp
        L.lwf_reader_read_dec_packet.argtypes = [vp, C.c_int, vp, sz, C.POINTER(sz)]
        L.lwf_reader_last_absgp.argtypes = [vp, C.POINTER(C.c_uint64)]
        L.lwf_reader_skip_samples_linear.argtypes = [vp, sz, C.c_int, vp, sz, C.POINTER(sz), C.POINTER(sz), C.POINTER(C.c_int)]
        L.lwf_reader_seek_absgp_pg.argtypes = [vp, C.c_uint64]
        L.lwf_batcher_create.argtypes = [vp, vp, C.c_int, C.POINTER(vp)]
        L.lwf_batcher_destroy.argtypes = [vp]
        L.lwf_batcher_destroy.restype = None
        L.lwf_batcher_set_entry.argtypes = [vp, C.c_int]
        L.lwf_batcher_add_headers.argtypes = [vp, vp, vp]
        L.lwf_headers_vq_capable.argtypes = [vp]
        L.lwf_packet_decode_vq.argtypes = [vp, C.c_char_p, sz, vp, vp, sz, C.POINTER(sz), vp, sz, C.POINTER(sz)]
        L.lwf_packet_decode_vq_ex.argtypes = [vp, C.c_char_p, sz, vp, vp, sz, C.POINTER(sz), vp, sz, C.POINTER(sz), C.c_int]
        L.lwf_batcher_decode.argtypes = [vp, C.POINTER(_StreamJob), sz, C.c_int, vp]
        L.lwf_batcher_submit.argtypes = [vp, C.POINTER(_StreamJob), sz, C.c_int, vp, C.c_int, C.POINTER(C.c_uint64)]
        L.lwf_batcher_last_timing.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.lwf_batcher_last_timing.restype = None
        L.lwf_readers_create.argtypes = [vp, C.c_int, C.POINTER(vp)]
        L.lwf_readers_destroy.argtypes = [vp]
        L.lwf_readers_destroy.restype = None
        L.lwf_readers_add.argtypes = [vp, C.c_char_p, sz, C.POINTER(C.c_uint32)]
        L.lwf_readers_headers.argtypes = [vp, C.c_uint32]
        L.lwf_readers_headers.restype = vp
        L.lwf_readers_last_absgp.argtypes = [vp, C.c_uint32, C.POINTER(C.c_uint64)]
        L.lwf_readers_setup_count.argtypes = [vp]
        L.lwf_readers_setup_count.restype = C.c_uint32
        L.lwf_readers_last_timing.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.lwf_readers_last_timing.restype = None
        L.lwf_readers_read.argtypes = [vp, C.POINTER(_ReadJob), sz, C.c_int, vp, C.c_int, C.POINTER(C.c_uint64)]
        L.lwf_readers_seek_absgp_pg.argtypes = [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), sz, C.POINTER(C.c_int32)]
        L.lwf_readers_skip_samples_linear.argtypes = [vp, C.POINTER(_SkipJob), sz, C.c_int, vp, C.c_int, C.POINTER(C.c_uint64)]
        L.lwf_debug_float32_unpack.argtypes = [C.c_uint32]
        L.lwf_debug_float32_unpack.restype = C.c_float
        L.lwf_debug_lookup1_values.argtypes = [C.c_uint32, C.c_uint16]
        L.lwf_debug_lookup1_values.restype = C.c_uint32
        L.lwf_debug_ilog.argtypes = [C.c_uint64]
        L.lwf_debug_ilog.restype = C.c_uint8
        L.lwf_debug_read_bits.argtypes = [C.c_char_p, sz, C.c_char_p, sz, C.POINTER(C.c_uint64)]
        L.lwf_debug_read_bits.restype = sz
        L.lwf_debug_huffman.argtypes = [C.c_char_p, sz, C.c_char_p, sz, cabi.u32p, sz, C.POINTER(sz)]
        _declared = True
    return L


class Headers:
    """The three parsed Vorbis headers."""

    def __init__(self, ident, comment, setup, _handle=None):
        self._own = _handle is None
        if _handle is None:
            h = C.c_void_p()
            rc = lib().lwf_headers_parse(ident, len(ident), comment, len(comment), setup, len(setup), C.byref(h))
            if rc:
                raise HeaderReadError(rc)
            _handle = h.value
        self._h = _handle
        info = Info()
        lib().lwf_headers_info(self._h, C.byref(info))
        self.info = info
        for f, _ in Info._fields_:
            setattr(self, f, getattr(info, f))

    def _str(self, index):
        n = lib().lwf_headers_comment(self._h, index, None, 0)
        buf = C.create_string_buffer(n + 1)
        lib().lwf_headers_comment(self._h, index, buf, n + 1)
        return buf.raw[:n].decode("utf-8")

    @property
    def vendor(self):
        return self._str(-1)

    @property
    def comment_list(self):
        out = []
        for i in range(self.n_comments):
            k, _, v = self._str(i).partition("=")
            out.append((k, v))
        return out

    def make_setup(self, ctx, floor0=False):
        """The device-side header constants (lwb_setup) for these headers; floor0: with the floor-0 descriptions that
        packets decoded with floor0_records=True need (lwf_headers_make_setup_floor0)."""
        h = C.c_void_p()
        fn = lib().lwf_headers_make_setup_floor0 if floor0 else lib().lwf_headers_make_setup
        ctx.check(fn(self._h, ctx._h, C.byref(h)))
        return Setup._adopt(ctx, h.value, self.audio_channels, self.blocksize_0, self.blocksize_1)

    def decode_packet(self, packet, floor0_records=False):
        """audio.rs:919-986: returns an api.DecodedPacket (mode, window flags, per-channel floors, residue).
        floor0_records: type-0 floors of order <= 63 come out as api.Floor0Record instead of dense curves."""
        Cn, n2max = self.audio_channels, (1 << self.blocksize_1) // 2
        kinds = np.zeros(Cn, np.uint8)
        ys = np.zeros((Cn, cabi.MAX_POSTS), np.uint32)
        dense = np.zeros((Cn, n2max), np.float32)
        res = np.zeros((Cn, n2max), np.float32)
        dp = _DecodedPacket()
        dp.floor_kind = kinds.ctypes.data_as(cabi.u8p)
        dp.floor1_y = ys.ctypes.data_as(cabi.u32p)
        dp.dense_floor = dense.ctypes.data_as(cabi.fp)
        dp.residue = res.ctypes.data_as(cabi.fp)
        rc = lib().lwf_packet_decode_ex(self._h, bytes(packet), len(packet), C.byref(dp), FLOOR0_RECORDS if floor0_records else 0)
        if rc == cabi.ERR_BAD_FORMAT:
            raise AudioReadError(rc)
        if rc:
            e = AudioReadError(rc)
            e.kind = {ERR_END_OF_PACKET: "EndOfPacket", ERR_AUDIO_IS_HEADER: "AudioIsHeader"}.get(rc, e.kind)
            raise e
        n2 = dp.n // 2
        floors = []
        flat_dense = dense.ravel()
        flat_res = res.ravel()
        for c in range(Cn):
            if kinds[c] == cabi.FLOOR_UNUSED:
                floors.append(None)
            elif kinds[c] == cabi.FLOOR_ONE:
                floors.append(ys[c].copy())
            elif kinds[c] == cabi.FLOOR_ZERO:
                floors.append(_record(ys[c]))
            else:
                floors.append(flat_dense[c * n2:(c + 1) * n2].copy())
        residue = flat_res[: Cn * n2].reshape(Cn, n2).copy()
        out = DecodedPacket(dp.mode_number, residue, floors, dp.prev_window_flag, dp.next_window_flag)
        out.blockflag, out.n = bool(dp.blockflag), dp.n
        return out

    def vq_capable(self):
        """True if LWB_ENTRY_VQ applies to this stream (lwf_headers_vq_capable)."""
        return bool(lib().lwf_headers_vq_capable(self._h))

    def decode_packet_vq(self, packet, floor0_records=False):
        """The same front half with the residue left as VQ runs: (DecodedPacket with a zero residue, runs, entries):
        runs a structured array (lwb_vq_run), entries the uint16 codebook entries they index."""
        Cn, n2max = self.audio_channels, (1 << self.blocksize_1) // 2
        kinds = np.zeros(Cn, np.uint8)
        ys = np.zeros((Cn, cabi.MAX_POSTS), np.uint32)
        dense = np.zeros((Cn, n2max), np.float32)
        dp = _DecodedPacket()
        dp.floor_kind = kinds.ctypes.data_as(cabi.u8p)
        dp.floor1_y = ys.ctypes.data_as(cabi.u32p)
        dp.dense_floor = dense.ctypes.data_as(cabi.fp)
        cap = len(packet) * 8 + 16
        runs, ents = np.zeros(cap, VQ_RUN_DTYPE), np.zeros(cap, np.uint16)
        n, ne = C.c_size_t(), C.c_size_t()
        rc = lib().lwf_packet_decode_vq_ex(self._h, bytes(packet), len(packet), C.byref(dp), runs.ctypes.data, cap, C.byref(n),
                                           ents.ctypes.data, cap, C.byref(ne), FLOOR0_RECORDS if floor0_records else 0)
        if rc == cabi.ERR_BAD_FORMAT:
            raise AudioReadError(rc)
        if rc:
            e = AudioReadError(rc)
            e.kind = {ERR_END_OF_PACKET: "EndOfPacket", ERR_AUDIO_IS_HEADER: "AudioIsHeader"}.get(rc, e.kind)
            raise e
        n2 = dp.n // 2
        floors = []
        flat_dense = dense.ravel()
        for c in range(Cn):
            if kinds[c] == cabi.FLOOR_UNUSED:
                floors.append(None)
            elif kinds[c] == cabi.FLOOR_ONE:
                floors.append(ys[c].copy())
            elif kinds[c] == cabi.FLOOR_ZERO:
                floors.append(_record(ys[c]))
            else:
                floors.append(flat_dense[c * n2:(c + 1) * n2].copy())
        out = DecodedPacket(dp.mode_number, np.zeros((Cn, n2), np.float32), floors, dp.prev_window_flag, dp.next_window_flag)
        out.blockflag, out.n = bool(dp.blockflag), dp.n
        return out, runs[: n.value].copy(), ents[: ne.value].copy()

    def decoded_sample_count(self, packet):
        n = C.c_size_t()
        rc = lib().lwf_decoded_sample_count(self._h, bytes(packet), len(packet), C.byref(n))
        if rc:
            raise AudioReadError(rc, "get_decoded_sample_count")
        return n.value

    def close(self):
        if self._h and self._own:
            lib().lwf_headers_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class OggPacket:
    def __init__(self, p):
        self.data = C.string_at(p.data, p.len) if p.len else b""
        self.stream_serial, self.absgp_page = p.stream_serial, p.absgp_page
        self.first_in_stream, self.last_in_stream = bool(p.first_in_stream), bool(p.last_in_stream)
        self.first_in_page, self.last_in_page = bool(p.first_in_page), bool(p.last_in_page)


class OggPacketReader:
    def __init__(self, data):
        self._data = bytes(data)
        h = C.c_void_p()
        rc = lib().lwf_ogg_open(self._data, len(self._data), C.byref(h))
        if rc:
            raise OggReadError("open: %d" % rc)
        self._h = h.value

    def read_packet(self):
        """Next packet or None at the end of the data."""
        p = _OggPacket()
        rc = lib().lwf_ogg_next_packet(self._h, C.byref(p))
        if rc == ERR_NO_MORE_PACKETS:
            return None
        if rc:
            raise OggReadError("framing error (%d)" % rc)
        return OggPacket(p)

    def close(self):
        if self._h:
            lib().lwf_ogg_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def read_headers(reader):
    """inside_ogg.rs:19-39 on an OggPacketReader: (Headers, stream_serial)."""
    pk = reader.read_packet()
    ident, serial = pk.data, pk.stream_serial
    pk = reader.read_packet()
    while pk.stream_serial != serial:
        pk = reader.read_packet()
    comment = pk.data
    pk = reader.read_packet()
    while pk.stream_serial != serial:
        pk = reader.read_packet()
    return Headers(ident, comment, pk.data), serial


class OggStreamReader:
    """inside_ogg.rs:60-227: ogg/vorbis bytes in, PCM packets out (synthesis on the GPU)."""

    def __init__(self, ctx, data):
        self.ctx = ctx
        self._data = bytes(data)
        h = C.c_void_p()
        rc = lib().lwf_reader_open(ctx._h, self._data, len(self._data), C.byref(h))
        if rc:
            if 16 <= rc <= 22:
                raise HeaderReadError(rc)
            if rc >= ERR_OGG:
                raise OggReadError("code %d" % rc)
            ctx.check(rc)
        self._h = h.value
        self._buf = None
        # more than one logical stream in the data: the next one may have any channel count / blocksize
        self._may_chain = self._data.count(b"OggS\x00\x02") > 1
        ctx._children.add(self)
        self._refresh()

    def _refresh(self):
        self.headers = Headers(None, None, None, _handle=lib().lwf_reader_headers(self._h))
        self.ident_hdr = self.headers

    def _read(self, fmt, dtype, interleaved, skip=None):
        total = 255 * 8192 if self._may_chain else self.headers.audio_channels << self.headers.blocksize_1
        if self._buf is None or self._buf.size < total or self._buf.dtype != dtype:
            self._buf = np.zeros(total, dtype)
        buf = self._buf
        n = C.c_size_t()
        if skip is None:
            rc = lib().lwf_reader_read_dec_packet(self._h, fmt, buf.ctypes.data, buf.size, C.byref(n))
        else:
            left, got = C.c_size_t(), C.c_int()
            rc = lib().lwf_reader_skip_samples_linear(self._h, skip, fmt, buf.ctypes.data, buf.size, C.byref(n), C.byref(left),
                                                      C.byref(got))
            self._skip_left = left.value
            if rc == 0 and not got.value:
                return None
        if rc == ERR_NO_MORE_PACKETS:
            return None
        e = read_error(self.ctx, rc)
        if e is not None:
            raise e
        if lib().lwf_reader_headers(self._h) != self.headers._h:
            self._refresh()                      # a chained stream started
        Cn = self.headers.audio_channels
        if interleaved:
            return buf[: n.value * Cn].copy()
        cap = buf.size // Cn
        return [buf[c * cap: c * cap + n.value].copy() for c in range(Cn)]

    def read_dec_packet(self):
        """Vec<Vec<i16>> or None"""
        return self._read(cabi.OUT_I16_PLANAR, np.int16, False)

    def read_dec_packet_itl(self):
        """interleaved Vec<i16> or None"""
        return self._read(cabi.OUT_I16_INTERLEAVED, np.int16, True)

    def read_dec_packet_f32(self):
        """read_dec_packet_generic::<Vec<Vec<f32>>>"""
        return self._read(cabi.OUT_F32_PLANAR, np.float32, False)

    def read_dec_packet_generic(self, sample="f32", interleaved=False):
        """inside_ogg.rs:191-205, read_dec_packet_generic::<S>: sample "f32" | "i16" | "f16" (numpy float16: the f32
        samples rounded to nearest even) | "i32" | "i24" (api.I24 elements); planar [channels] arrays or one interleaved
        array, or None at the end."""
        fmt, dt = sample_format(sample, interleaved)
        return self._read(fmt, dt, bool(interleaved))

    def skip_samples_linear(self, to_skip, sample="f32"):
        """inside_ogg.rs:244-283 -> (Option<S>, usize): (planar packet or None, samples left to skip inside it).  sample:
        "f32", "f16", "i32", "i24", else i16."""
        fmt, dt = sample_format(sample if sample in ("f32", "f16", "i32", "i24") else "i16")
        pck = self._read(fmt, dt, False, skip=int(to_skip))
        return pck, self._skip_left

    def seek_absgp_pg(self, absgp):
        """inside_ogg.rs:307-313: page-granular seek to a position <= absgp; resets cur_absgp and PreviousWindowRight."""
        rc = lib().lwf_reader_seek_absgp_pg(self._h, int(absgp))
        if rc >= ERR_OGG:
            raise OggReadError("code %d" % rc)
        self.ctx.check(rc)

    def get_last_absgp(self):
        v = C.c_uint64()
        return v.value if lib().lwf_reader_last_absgp(self._h, C.byref(v)) == 0 else None

    def close(self):
        if self._h:
            lib().lwf_reader_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


FLOOR0_RECORDS = 1           # LWF_DECODE_FLOOR0_RECORDS


def _record(row):
    """The api.Floor0Record in an LWB_FLOOR_ZERO floor1_y row: the amplitude and all 63 coefficient slots (those past the
    floor's order are zero, and the device does not read them)."""
    return Floor0Record(int(row[0]) | (int(row[1]) << 32), row[2:].view(np.float32).copy())


class StreamBatcher:
    """lwf_batcher: entropy-decode the packets of many streams on a host thread pool and synthesise them with one
    batched call per group of header sets (one group unless add_headers registered more).  jobs: list of
    (PreviousWindowRight, [packet bytes, ...]); job j's PCM lands in `pcm` behind the jobs before it, each taking its
    stream's output channels * stride elements (Setup.output_channels: audio_channels unless the setup has an output mix;
    out_offset = job index * channels * stride for one set of headers)."""

    def __init__(self, ctx, headers, threads=0, entry=cabi.ENTRY_RESIDUE, floor0=False):
        """floor0: type-0 floors travel as floor-0 records (lwf_batcher_set_floor0); the jobs' streams must then come from
        headers.make_setup(ctx, floor0=True)."""
        self.ctx, self.headers = ctx, headers
        h = C.c_void_p()
        ctx.check(lib().lwf_batcher_create(ctx._h, headers._h, threads, C.byref(h)))
        self._h = h.value
        self._sets = []
        ctx._children.add(self)
        if floor0:
            ctx.check(lib().lwf_batcher_set_floor0(self._h, 1))
        if entry != cabi.ENTRY_RESIDUE:        # LWB_ENTRY_VQ: VQ records instead of dense residue vectors cross the boundary
            rc = lib().lwf_batcher_set_entry(self._h, entry)
            if rc:
                raise AudioReadError(rc, "this stream does not qualify for LWB_ENTRY_VQ (lwf_headers_vq_capable)")

    def add_headers(self, headers, setup):
        """lwf_batcher_add_headers: the jobs of streams opened on `setup` (an api.Setup made from `headers`) are decoded
        with `headers`; both are kept alive with the batcher."""
        self.ctx.check(lib().lwf_batcher_add_headers(self._h, headers._h, setup._h))
        self._sets.append((headers, setup))

    def _jobs(self, jobs, stride):
        """The lwf_stream_job array of `jobs`, and the packet arrays it points to."""
        n = len(jobs)
        arr = (_StreamJob * n)()
        keep = []
        off = 0
        for j, (pwr, packets) in enumerate(jobs):
            pk = (C.c_char_p * len(packets))(*packets)
            ln = (C.c_size_t * len(packets))(*[len(p) for p in packets])
            keep.append((pk, ln))
            arr[j].stream = pwr._h
            arr[j].n_packets = len(packets)
            arr[j].packets = pk
            arr[j].lengths = ln
            arr[j].out_offset = off
            arr[j].out_stride = stride
            off += pwr.setup.output_channels * stride
        return arr, keep, n

    def _counters(self):
        e, s = C.c_double(), C.c_double()
        lib().lwf_batcher_last_timing(self._h, C.byref(e), C.byref(s))
        self.entropy_seconds, self.synthesis_seconds = e.value, s.value
        self.input_bytes = lib().lwf_batcher_last_input_bytes(self._h)

    def decode(self, jobs, pcm, stride, out_format=cabi.OUT_F32_PLANAR):
        self.prepared = self._jobs(jobs, stride)
        return self.run(pcm, out_format)

    def run(self, pcm, out_format=cabi.OUT_F32_PLANAR):
        """Decode the jobs of the last decode() again (same packets; benchmarking)."""
        arr, _, n = self.prepared
        self.ctx.check(lib().lwf_batcher_decode(self._h, arr, n, out_format, pcm.ctypes.data))
        self._counters()
        return _results(arr, n)

    def submit(self, jobs, pcm, stride, out_format=cabi.OUT_F32_PLANAR):
        """lwf_batcher_submit: entropy-decodes `jobs` (as decode()), queues their synthesis and returns an api.Ticket
        once it is queued; its wait() returns the job results [(n_samples, packets_done, status)], as run() does.  pcm: a
        page-locked numpy array (Context.host_alloc), a torch CUDA tensor or an integer device pointer; the memory space
        follows from it.  The streams may be submitted again at once; `pcm` holds the PCM once the ticket is done, and
        the ticket keeps it and the job arrays alive until then.  entropy_seconds / synthesis_seconds / input_bytes
        describe this submit."""
        addr, memory = _pcm_address(pcm)
        arr, keep, n = self._jobs(jobs, stride)
        t = C.c_uint64()
        self.ctx.check(lib().lwf_batcher_submit(self._h, arr, n, out_format, addr, memory, C.byref(t)))
        self._counters()
        return Ticket(self.ctx, t.value, (keep, pcm), lambda: _results(arr, n))

    def close(self):
        if self._h:
            lib().lwf_batcher_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _results(arr, n):
    return [(arr[j].n_samples, arr[j].packets_done, arr[j].status) for j in range(n)]


def _pcm_address(pcm):
    """(address, LWB_MEM_*) of a page-locked numpy array, a torch CUDA tensor or an integer device pointer."""
    if isinstance(pcm, np.ndarray):
        return pcm.ctypes.data, cabi.MEM_HOST
    if isinstance(pcm, int):
        return pcm, cabi.MEM_DEVICE
    if hasattr(pcm, "data_ptr") and getattr(pcm, "is_cuda", False):
        return pcm.data_ptr(), cabi.MEM_DEVICE
    raise TypeError("pcm: a page-locked numpy array, a torch CUDA tensor or an integer device pointer")


def read_error(ctx, rc):
    """The exception OggStreamReader raises for status `rc` of a packet (None for LWB_OK; LWF_ERR_NO_MORE_PACKETS, the
    end, is the caller's to handle)."""
    if rc == 0:
        return None
    if rc == cabi.ERR_BAD_FORMAT:
        return AudioReadError(rc)
    if rc in (ERR_END_OF_PACKET, ERR_AUDIO_IS_HEADER):
        e = AudioReadError(rc)
        e.kind = {ERR_END_OF_PACKET: "EndOfPacket", ERR_AUDIO_IS_HEADER: "AudioIsHeader"}[rc]
        return e
    if 16 <= rc <= 23:               # the headers of a chained stream (inside_ogg.rs:118-137): VorbisError::BadHeader
        return HeaderReadError(rc)
    if rc >= ERR_OGG:
        return OggReadError("code %d" % rc)
    try:
        ctx.check(rc)
    except Exception as e:      # noqa: BLE001 -- the exception object is the result
        return e
    return None


class ReadResult:
    """One job of OggStreamReaders.read: the packets it returned (n_packets, and packet_samples, the samples each wrote),
    n_samples per channel written at out_offset (planar: channel c at out_offset + c * out_stride; interleaved: `channels`
    samples per frame), and how the reader stopped: status (LWB_OK or the code the single reader's next call returned),
    ended (no packet left) and next_chained (the reader stands at a new logical stream)."""

    def __init__(self, job, packet_samples):
        for f, _ in _ReadJob._fields_:
            if f not in ("packet_samples", "reserved"):
                setattr(self, f, getattr(job, f))
        self.next_chained, self.ended = bool(self.next_chained), bool(self.ended)
        self.packet_samples = packet_samples[: self.n_packets].copy()

    def __repr__(self):
        return ("ReadResult(reader=%d, n_packets=%d, n_samples=%d, channels=%d, status=%d, ended=%s, next_chained=%s)" %
                (self.reader, self.n_packets, self.n_samples, self.channels, self.status, self.ended, self.next_chained))


class SkipResult:
    """One job of OggStreamReaders.skip_samples_linear: got_packet (a packet was returned), its n_samples per channel at
    out_offset (planar: channel c at out_offset + c * out_stride; interleaved: `channels` samples per frame),
    left_to_skip, the channel count of the stream the reader stands in, and status (LWB_OK or the code the single
    reader's call returned)."""

    def __init__(self, job):
        for f, _ in _SkipJob._fields_:
            if f != "reserved":
                setattr(self, f, getattr(job, f))
        self.got_packet = bool(self.got_packet)

    def __repr__(self):
        return ("SkipResult(reader=%d, got_packet=%s, n_samples=%d, left_to_skip=%d, channels=%d, status=%d)" %
                (self.reader, self.got_packet, self.n_samples, self.left_to_skip, self.channels, self.status))


def _packet_pcm(pcm, offset, stride, channels, s0, n, interleaved):
    """A copy of samples [s0, s0 + n) of the job PCM at `offset` in `pcm`, in the form OggStreamReader returns a
    packet: one interleaved array, or a list of per-channel arrays (planes `stride` apart)"""
    if interleaved:
        return pcm[offset + s0 * channels: offset + (s0 + n) * channels].copy()
    return [pcm[offset + c * stride + s0: offset + c * stride + s0 + n].copy() for c in range(channels)]


def _stream_shapes(data):
    """(channels, blocksize_0, blocksize_1) of every logical stream of Ogg Vorbis bytes whose first page holds a Vorbis
    ident header, from the beginning-of-stream pages; the walk stops at the first page it cannot parse."""
    out, at = [], 0
    while at + 27 <= len(data) and data[at:at + 4] == b"OggS":
        nseg = data[at + 26]
        body = at + 27 + nseg
        end = body + sum(data[at + 27: body])
        if end > len(data):
            break
        first = data[body: body + 30]
        if data[at + 5] & 2 and len(first) == 30 and first[:7] == b"\x01vorbis":
            out.append((first[11], first[28] & 15, first[28] >> 4))
        at = end
    return out


class OggStreamReaders:
    """Many OggStreamReaders on one context (lwf_readers): read() advances any of them by up to max_packets audio packets
    in one call -- de-paging and entropy decode on a host thread pool, synthesis as one batch per channel count and
    blocksize pair on the fused kernels -- and each returns exactly what OggStreamReader.read_dec_packet_generic returns,
    packet for packet.  seek_absgp_pg() and skip_samples_linear() do the single reader's seek and skip for many readers
    in one call, holding each to what OggStreamReader returns too.  Readers whose ident and setup headers are byte-equal
    share one device setup."""

    def __init__(self, ctx, threads=0):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.check(lib().lwf_readers_create(ctx._h, threads, C.byref(h)))
        self._h = h.value
        self._data = []                          # the bytes of each reader: lwf_readers_add does not copy them
        self._shapes = []                        # (channels, blocksize_0, blocksize_1) of each file's logical streams
        self._headers = {}
        ctx._children.add(self)

    def add(self, data):
        """A reader over `data` (OggStreamReader(ctx, data)): its headers are read now.  Returns its index."""
        data = bytes(data)
        i = C.c_uint32()
        rc = lib().lwf_readers_add(self._h, data, len(data), C.byref(i))
        if rc:
            e = read_error(self.ctx, rc)
            raise e if e is not None else AudioReadError(rc)
        self._data.append(data)
        self._shapes.append(_stream_shapes(data))       # the bytes never change: walked once, for skip_room
        return i.value

    def stride(self, index, max_packets):
        """The least planar stride of a job of max_packets packets of reader `index` (lwf_readers_read refuses a smaller
        one): max_packets * blocksize_1 / 2 + (blocksize_1 - blocksize_0) / 4 of its stream."""
        h = self.headers(index)
        n1, n0 = 1 << h.blocksize_1, 1 << h.blocksize_0
        return max_packets * n1 // 2 + (n1 - n0) // 4 if max_packets else 0

    def __len__(self):
        return len(self._data)

    def headers(self, index):
        """Headers of the stream reader `index`'s next packet belongs to (after a job with next_chained: the new one's)."""
        h = lib().lwf_readers_headers(self._h, index)
        if not h:
            raise IndexError(index)
        if self._headers.get(index, (None,))[0] != h:
            self._headers[index] = (h, Headers(None, None, None, _handle=h))
        return self._headers[index][1]

    def get_last_absgp(self, index):
        v = C.c_uint64()
        return v.value if lib().lwf_readers_last_absgp(self._h, index, C.byref(v)) == 0 else None

    @property
    def setup_count(self):
        """Distinct (ident, setup) header pairs among the streams opened: one device setup each."""
        return lib().lwf_readers_setup_count(self._h)

    def _queue(self, call, arr, fmt, addr, memory, result, keep):
        """call (lwf_readers_read or lwf_readers_skip_samples_linear) on the job array arr; records its timings and
        returns an api.Ticket that keeps `keep` alive, with results [result(j)] for every job j"""
        t = C.c_uint64()
        self.ctx.check(call(self._h, arr, len(arr), fmt, addr, memory, C.byref(t)))
        p, e, s = C.c_double(), C.c_double(), C.c_double()
        lib().lwf_readers_last_timing(self._h, C.byref(p), C.byref(e), C.byref(s))
        self.paging_seconds, self.entropy_seconds, self.synthesis_seconds = p.value, e.value, s.value
        results = [result(j) for j in range(len(arr))]
        ticket = Ticket(self.ctx, t.value, keep, lambda: results)
        ticket.results = results
        return ticket

    def read(self, jobs, pcm, stride, sample="f32", interleaved=False):
        """lwf_readers_read.  jobs: [(reader index, max_packets)], each reader at most once.  Job j's PCM lands in `pcm`
        behind the jobs before it, each taking its reader's channels * stride elements (planar: channel c at
        offset + c * stride; stride >= self.stride(index, max_packets) of every job).  pcm: a page-locked numpy array
        (Context.host_alloc), a torch CUDA tensor or an integer device pointer, as for StreamBatcher.submit.  Returns an
        api.Ticket; its results ([ReadResult], `results` and what wait() returns) are known at once, its PCM once it is
        done, and it keeps `pcm` alive until then.  paging_seconds, entropy_seconds and synthesis_seconds describe this
        read (lwf_readers_last_timing)."""
        fmt, _ = sample_format(sample, interleaved)
        addr, memory = _pcm_address(pcm)
        n = len(jobs)
        arr = (_ReadJob * n)()
        counts = []
        off = 0
        for j, (index, max_packets) in enumerate(jobs):
            ps = np.zeros(max(1, max_packets), np.uint32)
            counts.append(ps)
            arr[j].reader, arr[j].max_packets = index, max_packets
            arr[j].out_offset, arr[j].out_stride = off, stride
            arr[j].packet_samples = ps.ctypes.data_as(cabi.u32p)
            off += self.headers(index).audio_channels * stride
        return self._queue(lib().lwf_readers_read, arr, fmt, addr, memory, lambda j: ReadResult(arr[j], counts[j]),
                           (arr, counts, pcm))

    def read_dec_packets(self, indices, max_packets, sample="f32", interleaved=False):
        """read() into page-locked host memory and wait: per reader, the packets it returned, each in the form
        OggStreamReader.read_dec_packet_generic returns it (planar: a list of per-channel arrays; interleaved: one array),
        then None if it reached the end, or the exception the single reader's next call would have raised."""
        fmt, dt = sample_format(sample, interleaved)
        if not indices:
            return []
        stride = max([1] + [self.stride(i, max_packets) for i in indices])
        total = sum(self.headers(i).audio_channels for i in indices) * stride
        pcm = self.ctx.host_alloc(max(1, total), dt)
        results = self.read([(i, max_packets) for i in indices], pcm, stride, sample, interleaved).wait()
        out = []
        for r in results:
            pkts, s0 = [], 0
            for n in map(int, r.packet_samples):
                pkts.append(_packet_pcm(pcm, r.out_offset, stride, r.channels, s0, n, interleaved))
                s0 += n
            if r.status:
                pkts.append(read_error(self.ctx, r.status))
            elif r.ended:
                pkts.append(None)
            out.append(pkts)
        return out

    def seek_absgp_pg(self, indices, absgps):
        """lwf_readers_seek_absgp_pg: OggStreamReader.seek_absgp_pg(absgps[k]) on reader indices[k], each reader at most
        once; the pages are walked on the host thread pool and nothing is queued on the GPU.  Returns per reader None, or
        the exception the single reader would have raised (its position is then unchanged)."""
        n = len(indices)
        if not n:
            return []
        idx = (C.c_uint32 * n)(*indices)
        gps = (C.c_uint64 * n)(*[int(g) for g in absgps])
        st = (C.c_int32 * n)()
        self.ctx.check(lib().lwf_readers_seek_absgp_pg(self._h, idx, gps, n, st))
        return [read_error(self.ctx, rc) for rc in st]

    def skip_room(self, index):
        """(channels, stride): the room a skip job of reader `index` takes -- the most channels of any logical stream of
        its file, and the planar stride that one packet of any of them needs (blocksize_1 / 2 + (blocksize_1 -
        blocksize_0) / 4), so that a skip into a chained stream fits too."""
        h = self.headers(index)
        shapes = self._shapes[index] + [(h.audio_channels, h.blocksize_0, h.blocksize_1)]
        return (max(c for c, _, _ in shapes), max((1 << b1) // 2 + ((1 << b1) - (1 << b0)) // 4 for _, b0, b1 in shapes))

    def skip_samples_linear(self, jobs, pcm, stride, sample="f32", interleaved=False):
        """lwf_readers_skip_samples_linear.  jobs: [(reader index, to_skip)], each reader at most once.  Job j's target
        packet lands in `pcm` behind the jobs before it, each taking skip_room(index)[0] * stride elements (planar: channel
        c at offset + c * stride; stride >= skip_room(index)[1] of every job).  pcm as for read().  Returns an api.Ticket
        whose results ([SkipResult], `results` and what wait() returns) are known at once and its PCM once it is done;
        paging_seconds (the walk), entropy_seconds and synthesis_seconds describe this call."""
        fmt, _ = sample_format(sample, interleaved)
        addr, memory = _pcm_address(pcm)
        n = len(jobs)
        arr = (_SkipJob * n)()
        off = 0
        for j, (index, to_skip) in enumerate(jobs):
            room = self.skip_room(index)[0]
            arr[j].reader, arr[j].to_skip, arr[j].out_channels = index, int(to_skip), room
            arr[j].out_offset, arr[j].out_stride = off, stride
            off += room * stride
        return self._queue(lib().lwf_readers_skip_samples_linear, arr, fmt, addr, memory, lambda j: SkipResult(arr[j]),
                           (arr, pcm))

    def skip_samples_linear_dec(self, indices, to_skip, sample="f32", interleaved=False):
        """skip_samples_linear() into page-locked host memory and wait: per reader what OggStreamReader.skip_samples_linear
        returns -- (packet or None, left_to_skip), the packet planar (a list of per-channel arrays) or interleaved (one
        array) -- or the exception it would have raised.  to_skip: one count for every reader, or one per reader."""
        fmt, dt = sample_format(sample, interleaved)
        if not indices:
            return []
        counts = list(to_skip) if hasattr(to_skip, "__len__") else [to_skip] * len(indices)
        rooms = [self.skip_room(i) for i in indices]
        stride = max(s for _, s in rooms)
        pcm = self.ctx.host_alloc(max(1, sum(c for c, _ in rooms) * stride), dt)
        out = []
        for r in self.skip_samples_linear(list(zip(indices, counts)), pcm, stride, sample, interleaved).wait():
            if r.status:
                out.append(read_error(self.ctx, r.status))
            elif not r.got_packet:
                out.append((None, r.left_to_skip))
            else:
                out.append((_packet_pcm(pcm, r.out_offset, stride, r.channels, 0, r.n_samples, interleaved), r.left_to_skip))
        return out

    def close(self):
        if self._h:
            lib().lwf_readers_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
