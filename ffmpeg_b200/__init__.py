"""ffmpeg_b200 — H100-native (sm_90a) replacements for FFmpeg's data-parallel DSP hot paths.

The product is the C-ABI shared library libb200dsp.so (include/b200dsp.h); this package is the thin host-side mirror
of the reference interfaces used by the tests and the benchmark.  Importing the package does not load the library;
the first call does, and it raises if the library was not built or no GPU is usable (there is no CPU fallback).
"""
from ._lib import B200Error, SO_PATH, lib  # noqa: F401
from .device import Device, launch_count  # noqa: F401
from . import swscale, idctdsp, fdctdsp, me_cmp, pel, tx, mpegvideo, float_dsp, hevcdsp, vp9dsp, vp8dsp, vc1dsp  # noqa: F401

__all__ = ["B200Error", "Device", "launch_count", "swscale", "idctdsp", "fdctdsp", "me_cmp", "pel", "tx", "mpegvideo", "float_dsp", "hevcdsp", "vp9dsp", "vp8dsp", "vc1dsp", "lib", "SO_PATH"]
