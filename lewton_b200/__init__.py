"""lewton_b200 -- H100-native Vorbis packet-synthesis back-end (the dense half of lewton's
audio::read_audio_packet*), as a C-ABI shared library plus this thin Python mirror.

Importing the package loads nothing; the first call into `lewton_b200.api` loads
lewton_b200/liblewton_b200.so and raises if it is absent (no CPU fallback).
"""
from . import _cabi  # noqa: F401
from .api import (AudioReadError, Batch, ChainSpec, Context, DecodedPacket, Floor0Record, FloorTypeOne, FloorTypeZero, Mapping,  # noqa: F401
                  ModeInfo, PreviousWindowRight, Setup, StateSlot, Ticket, VorbisError, debug_taps, decode_chains, decode_spectrum,
                  generate_tables, get_decoded_sample_count, i24_to_i32, mix_mono, mix_select, mix_wav_order, read_audio_packet,
                  read_audio_packet_generic, state_offsets)

__all__ = ["AudioReadError", "Batch", "ChainSpec", "Context", "DecodedPacket", "Floor0Record", "FloorTypeOne", "FloorTypeZero", "Mapping",
           "ModeInfo", "PreviousWindowRight", "Setup", "StateSlot", "Ticket", "VorbisError", "debug_taps", "decode_chains",
           "decode_spectrum", "generate_tables", "get_decoded_sample_count", "i24_to_i32", "mix_mono", "mix_select", "mix_wav_order",
           "read_audio_packet", "read_audio_packet_generic", "state_offsets"]
