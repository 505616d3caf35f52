"""A ctypes binding to the H.264 decoder of the libavcodec that the opencv-python wheel bundles: access units in, raw
Y / Cb / Cr planes out, with no colour conversion in between.  H.264 defines decoding exactly, so these planes are what
every conforming decoder outputs.

Only the fields the binding touches are read, at the offsets of the libavcodec 62 / libavutil 60 ABI; ``decoder()``
checks those versions and returns None when the library is absent or of another major version."""
from __future__ import annotations

import ctypes as C
import glob
import os
from typing import List, Optional, Tuple

import numpy as np

AVCODEC_MAJOR, AVUTIL_MAJOR = 62, 60
_PACKET_DATA = 24                       # AVPacket: buf, pts, dts, then data
_FRAME_LINESIZE = 64                    # AVFrame: data[8], then linesize[8]
_FRAME_WIDTH = 104                      # ... extended_data, then width, height
_EAGAIN = -11

_libs = None


def _load():
    global _libs
    if _libs is not None:
        return _libs or None
    _libs = False
    try:
        import cv2
    except ImportError:
        return None
    found = glob.glob(os.path.join(os.path.dirname(cv2.__file__), "..", "opencv_python*.libs"))
    if not found:
        return None

    def lib(name):
        paths = glob.glob(os.path.join(found[0], name + "-*.so*"))
        return C.CDLL(paths[0], mode=C.RTLD_GLOBAL) if paths else None
    util, codec = lib("libavutil"), None
    if util is not None and lib("libswresample") is not None:
        codec = lib("libavcodec")
    if codec is None:
        return None
    codec.avcodec_version.restype = C.c_uint
    util.avutil_version.restype = C.c_uint
    if codec.avcodec_version() >> 16 != AVCODEC_MAJOR or util.avutil_version() >> 16 != AVUTIL_MAJOR:
        return None
    vp = C.c_void_p
    for fn in ("avcodec_find_decoder_by_name", "avcodec_alloc_context3", "av_packet_alloc"):
        getattr(codec, fn).restype = vp
    codec.avcodec_find_decoder_by_name.argtypes = [C.c_char_p]
    codec.avcodec_alloc_context3.argtypes = [vp]
    codec.avcodec_open2.argtypes = [vp, vp, vp]
    codec.av_new_packet.argtypes = [vp, C.c_int]
    codec.avcodec_send_packet.argtypes = [vp, vp]
    codec.avcodec_receive_frame.argtypes = [vp, vp]
    codec.av_packet_unref.argtypes = [vp]
    codec.av_packet_free.argtypes = [C.POINTER(vp)]
    codec.avcodec_free_context.argtypes = [C.POINTER(vp)]
    util.av_frame_alloc.restype = vp
    util.av_frame_unref.argtypes = [vp]
    util.av_frame_free.argtypes = [C.POINTER(vp)]
    _libs = (codec, util)
    return _libs


def available() -> bool:
    return _load() is not None


def decode(access_units: List[bytes]) -> List[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
    """Decodes an Annex B H.264 stream given as one packet per access unit; returns (Y, Cb, Cr) uint8 planes per frame
    (4:2:0).  Raises RuntimeError if the library is missing or refuses the stream."""
    libs = _load()
    if libs is None:
        raise RuntimeError("libavcodec (opencv-python's bundled copy, ABI 62) is not available")
    codec, util = libs
    dec = codec.avcodec_find_decoder_by_name(b"h264")
    ctx = C.c_void_p(codec.avcodec_alloc_context3(dec))
    pkt = C.c_void_p(codec.av_packet_alloc())
    frame = C.c_void_p(util.av_frame_alloc())
    out = []
    try:
        if codec.avcodec_open2(ctx, dec, None) < 0:
            raise RuntimeError("avcodec_open2 failed")

        def drain():
            while True:
                rc = codec.avcodec_receive_frame(ctx, frame)
                if rc < 0:
                    return
                out.append(_planes(frame.value))
                util.av_frame_unref(frame)

        for au in access_units:
            if codec.av_new_packet(pkt, len(au)) < 0:
                raise RuntimeError("av_new_packet failed")
            data = C.cast(pkt.value + _PACKET_DATA, C.POINTER(C.c_void_p))[0]
            C.memmove(data, au, len(au))
            rc = codec.avcodec_send_packet(ctx, pkt)
            codec.av_packet_unref(pkt)
            if rc < 0 and rc != _EAGAIN:
                raise RuntimeError(f"avcodec_send_packet refused access unit {len(out)}: {rc}")
            drain()
        codec.avcodec_send_packet(ctx, None)
        drain()
    finally:
        util.av_frame_free(C.byref(frame))
        codec.av_packet_free(C.byref(pkt))
        codec.avcodec_free_context(C.byref(ctx))
    return out


def _planes(frame: int):
    ptrs = C.cast(frame, C.POINTER(C.c_void_p))
    ls = C.cast(frame + _FRAME_LINESIZE, C.POINTER(C.c_int))
    wh = C.cast(frame + _FRAME_WIDTH, C.POINTER(C.c_int))
    w, h = wh[0], wh[1]

    def plane(i, ph, pw):
        return np.stack([np.frombuffer(C.string_at(ptrs[i] + r * ls[i], pw), np.uint8) for r in range(ph)])
    return plane(0, h, w), plane(1, h // 2, w // 2), plane(2, h // 2, w // 2)


def decoder_version() -> Optional[int]:
    libs = _load()
    return None if libs is None else libs[0].avcodec_version()
