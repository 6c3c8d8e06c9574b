"""
tests/refheif_seq.py -- TEST INFRASTRUCTURE ONLY: ctypes access to the image-sequence C API of the UNMODIFIED reference
libheif (api/libheif/heif_sequences.h), on top of oracle/refheif.py: write a visual sequence track, decode it with
heif_track_decode_next_image, and read its raw samples with heif_track_get_next_raw_sequence_sample.

Like oracle/refheif.py it loads libheif_ref.so with RTLD_GLOBAL, so only use it in processes that never import torch.
"""
import ctypes as C
import struct

import numpy as np

from oracle import refheif as rh

ERROR_END_OF_SEQUENCE = 13
TRACK_TYPE_IMAGE_SEQUENCE = int.from_bytes(b"pict", "big")
COLORSPACE_UNDEFINED, CHROMA_UNDEFINED = 99, 99
CHANNEL_ALPHA = 6

_ready = False


class SecurityLimits(C.Structure):          # heif_security_limits up to max_total_memory (heif_security.h:37-64)
    _fields_ = [("version", C.c_uint8), ("max_image_size_pixels", C.c_uint64), ("max_number_of_tiles", C.c_uint64),
                ("max_bayer_pattern_pixels", C.c_uint32), ("max_items", C.c_uint32), ("max_color_profile_size", C.c_uint32),
                ("max_memory_block_size", C.c_uint64), ("max_components", C.c_uint32), ("max_iloc_extents_per_item", C.c_uint32),
                ("max_size_entity_group", C.c_uint32), ("max_children_per_box", C.c_uint32), ("max_total_memory", C.c_uint64)]


def load():
    """refheif.load() plus the signatures of the sequence entry points."""
    global _ready
    h = rh.load()
    if _ready:
        return h
    E = rh.Err
    sig = {
        "heif_track_options_alloc": (C.c_void_p, []),
        "heif_track_options_release": (None, [C.c_void_p]),
        "heif_track_options_set_timescale": (None, [C.c_void_p, C.c_uint32]),
        "heif_sequence_encoding_options_alloc": (C.c_void_p, []),
        "heif_sequence_encoding_options_release": (None, [C.c_void_p]),
        "heif_context_set_sequence_timescale": (None, [C.c_void_p, C.c_uint32]),
        "heif_context_set_number_of_sequence_repetitions": (None, [C.c_void_p, C.c_uint32]),
        "heif_context_add_visual_sequence_track": (E, [C.c_void_p, C.c_uint16, C.c_uint16, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
        "heif_image_set_duration": (None, [C.c_void_p, C.c_uint32]),
        "heif_image_get_duration": (C.c_uint32, [C.c_void_p]),
        "heif_track_encode_sequence_image": (E, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
        "heif_track_encode_end_of_sequence": (E, [C.c_void_p, C.c_void_p]),
        "heif_track_release": (None, [C.c_void_p]),
        "heif_context_has_sequence": (C.c_int, [C.c_void_p]),
        "heif_context_number_of_sequence_tracks": (C.c_int, [C.c_void_p]),
        "heif_context_get_track_ids": (None, [C.c_void_p, C.POINTER(C.c_uint32)]),
        "heif_context_get_track": (C.c_void_p, [C.c_void_p, C.c_uint32]),
        "heif_track_get_track_handler_type": (C.c_uint32, [C.c_void_p]),
        "heif_track_get_timescale": (C.c_uint32, [C.c_void_p]),
        "heif_track_has_alpha_channel": (C.c_int, [C.c_void_p]),
        "heif_track_get_image_resolution": (E, [C.c_void_p, C.POINTER(C.c_uint16), C.POINTER(C.c_uint16)]),
        "heif_track_decode_next_image": (E, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p]),
        "heif_track_get_next_raw_sequence_sample": (E, [C.c_void_p, C.POINTER(C.c_void_p)]),
        "heif_raw_sequence_sample_release": (None, [C.c_void_p]),
        "heif_raw_sequence_sample_get_data": (C.POINTER(C.c_uint8), [C.c_void_p, C.POINTER(C.c_size_t)]),
        "heif_raw_sequence_sample_get_duration": (C.c_uint32, [C.c_void_p]),
        "heif_image_get_colorspace": (C.c_int, [C.c_void_p]),
        "heif_image_get_chroma_format": (C.c_int, [C.c_void_p]),
        "heif_image_has_channel": (C.c_int, [C.c_void_p, C.c_int]),
        "heif_image_get_bits_per_pixel_range": (C.c_int, [C.c_void_p, C.c_int]),
        "heif_context_get_security_limits": (C.POINTER(SecurityLimits), [C.c_void_p]),
    }
    for name, (res, args) in sig.items():
        f = getattr(h, name)
        f.restype, f.argtypes = res, args
    _ready = True
    return h


class SequenceError(RuntimeError):
    def __init__(self, err, what):
        self.code, self.sub = err.code, err.sub
        super().__init__(f"libheif error {err.code}/{err.sub} {what}: {(err.msg or b'').decode(errors='replace')}")


def _check(err, what):
    if err.code != 0:
        raise SequenceError(err, what)


def new_encoder(quality=60, params=None):
    """The registered HEVC encoder of highest priority with the given quality and integer parameters (release with
    heif_encoder_release)."""
    h = load()
    ctx = h.heif_context_alloc()
    enc = C.c_void_p()
    try:
        rh.check(h.heif_context_get_encoder_for_format(ctx, rh.COMPRESSION_HEVC, C.byref(enc)), "get_encoder_for_format")
        rh.check(h.heif_encoder_set_lossy_quality(enc, quality))
        for k, v in (params or {}).items():
            rh.check(h.heif_encoder_set_parameter_integer(enc, k.encode(), int(v)), k)
    finally:
        h.heif_context_free(ctx)
    return enc


def write_sequence(path, images, quality=60, params=None, timescale=1000, durations=None, repetitions=None, encoder=None):
    """heif_context_add_visual_sequence_track ('pict', the given timescale), heif_image_set_duration, one
    heif_track_encode_sequence_image per image (heif_image pointers), heif_track_encode_end_of_sequence, write the file.
    The HEVC encoder is `encoder` (kept) or a new_encoder(quality, params) (released).  Raises SequenceError (with .code /
    .sub) on a refusal."""
    h = load()
    ctx = h.heif_context_alloc()
    own = encoder is None
    enc, track, topts, sopts = (new_encoder(quality, params) if own else encoder), C.c_void_p(), None, None
    try:
        if repetitions is not None:
            h.heif_context_set_number_of_sequence_repetitions(ctx, repetitions)
        topts = h.heif_track_options_alloc()
        h.heif_track_options_set_timescale(topts, timescale)
        sopts = h.heif_sequence_encoding_options_alloc()
        hh, ww = _image_size(images[0])
        _check(h.heif_context_add_visual_sequence_track(ctx, ww, hh, TRACK_TYPE_IMAGE_SEQUENCE, topts, sopts, C.byref(track)), "add_visual_sequence_track")
        for k, img in enumerate(images):
            h.heif_image_set_duration(img, durations[k] if durations else 1)
            _check(h.heif_track_encode_sequence_image(track, img, enc, sopts), f"encode_sequence_image (frame {k})")
        _check(h.heif_track_encode_end_of_sequence(track, enc), "encode_end_of_sequence")
        rh.check(h.heif_context_write_to_file(ctx, path.encode()), "write")
    finally:
        if track:
            h.heif_track_release(track)
        if sopts:
            h.heif_sequence_encoding_options_release(sopts)
        if topts:
            h.heif_track_options_release(topts)
        if own and enc:
            h.heif_encoder_release(enc)
        h.heif_context_free(ctx)


def _image_size(img):
    h = load()
    for ch in (rh.CHANNEL_Y, rh.CHANNEL_INTERLEAVED):
        w = h.heif_image_get_width(img, ch)
        if w > 0:
            return h.heif_image_get_height(img, ch), w
    raise ValueError("image has neither a Y nor an interleaved plane")


def _open(path):
    h = load()
    ctx = h.heif_context_alloc()
    rh.check(h.heif_context_read_from_file(ctx, path.encode(), None), "read")
    return ctx


def _tracks(h, ctx):
    n = h.heif_context_number_of_sequence_tracks(ctx)
    ids = (C.c_uint32 * max(n, 1))()
    h.heif_context_get_track_ids(ctx, ids)
    return [int(ids[i]) for i in range(n)]


def track_info(path):
    """Tracks of the file: [{id, handler, timescale, has_alpha, width, height}], first visual track first."""
    h = load()
    ctx = _open(path)
    out = []
    try:
        for tid in _tracks(h, ctx):
            t = h.heif_context_get_track(ctx, tid)
            w, hh = C.c_uint16(), C.c_uint16()
            e = h.heif_track_get_image_resolution(t, C.byref(w), C.byref(hh))
            out.append(dict(id=tid, handler=int(h.heif_track_get_track_handler_type(t)).to_bytes(4, "big").decode(errors="replace"),
                            timescale=int(h.heif_track_get_timescale(t)), has_alpha=bool(h.heif_track_has_alpha_channel(t)),
                            width=int(w.value) if e.code == 0 else None, height=int(hh.value) if e.code == 0 else None))
            h.heif_track_release(t)
    finally:
        h.heif_context_free(ctx)
    return out


def _planes(img):
    """The planes of a decoded heif_image as numpy arrays: {'interleaved'} or {'y', 'cb', 'cr', 'alpha'} (those present)."""
    h = load()
    out = {}
    for name, ch in (("y", rh.CHANNEL_Y), ("cb", rh.CHANNEL_CB), ("cr", rh.CHANNEL_CR), ("alpha", CHANNEL_ALPHA),("interleaved", rh.CHANNEL_INTERLEAVED)):
        if not h.heif_image_has_channel(img, ch):
            continue
        st = C.c_int()
        p = h.heif_image_get_plane_readonly(img, ch, C.byref(st))
        w, hh = h.heif_image_get_width(img, ch), h.heif_image_get_height(img, ch)
        bpp = h.heif_image_get_bits_per_pixel_range(img, ch)
        if ch == rh.CHANNEL_INTERLEAVED:
            nch = {rh.CHROMA_INTERLEAVED_RGB: 3, rh.CHROMA_INTERLEAVED_RGBA: 4}[h.heif_image_get_chroma_format(img)]
            out[name] = np.ctypeslib.as_array(p, shape=(hh, st.value))[:, :w * nch].copy().reshape(hh, w, nch)
        else:
            bps = 2 if bpp > 8 else 1
            a = np.ctypeslib.as_array(p, shape=(hh, st.value))[:, :w * bps].copy()
            out[name] = a.view(np.uint16) if bps == 2 else a
    return out


def decode_track(path, colorspace=COLORSPACE_UNDEFINED, chroma=CHROMA_UNDEFINED, decoder_id=None, max_calls=10000, max_total_memory=None):
    """heif_track_decode_next_image on the first visual track until it reports the end of the sequence (or max_calls calls),
    optionally with the context's max_total_memory security limit set.  Returns a list with one entry per call that did not
    end the sequence: ('ok', planes, duration) or ('error', code, message)."""
    h = load()
    ctx = _open(path)
    if max_total_memory is not None:
        lim = h.heif_context_get_security_limits(ctx).contents
        assert lim.version >= 2, lim.version
        lim.max_total_memory = max_total_memory
    t = h.heif_context_get_track(ctx, 0)
    if not t:
        h.heif_context_free(ctx)
        raise RuntimeError("no visual track")
    opts = h.heif_decoding_options_alloc()
    keep = decoder_id.encode() if decoder_id else None
    if keep:
        opts.contents.decoder_id = keep
    out = []
    try:
        for _ in range(max_calls):
            img = C.c_void_p()
            e = h.heif_track_decode_next_image(t, C.byref(img), colorspace, chroma, C.cast(opts, C.c_void_p))
            if e.code == ERROR_END_OF_SEQUENCE:
                break
            if e.code != 0:
                out.append(("error", int(e.code), (e.msg or b"").decode(errors="replace")))
                continue
            out.append(("ok", _planes(img), int(h.heif_image_get_duration(img))))
            h.heif_image_release(img)
    finally:
        h.heif_decoding_options_free(opts)
        h.heif_track_release(t)
        h.heif_context_free(ctx)
    return out


def raw_samples(path, track_id=0):
    """Every raw sample of a track (first visual track by default): [(bytes, duration)]."""
    h = load()
    ctx = _open(path)
    t = h.heif_context_get_track(ctx, track_id)
    out = []
    try:
        while True:
            s = C.c_void_p()
            e = h.heif_track_get_next_raw_sequence_sample(t, C.byref(s))
            if e.code == ERROR_END_OF_SEQUENCE:
                break
            rh.check(e, "get_next_raw_sequence_sample")
            n = C.c_size_t()
            p = h.heif_raw_sequence_sample_get_data(s, C.byref(n))
            out.append((C.string_at(p, n.value), int(h.heif_raw_sequence_sample_get_duration(s))))
            h.heif_raw_sequence_sample_release(s)
    finally:
        h.heif_track_release(t)
        h.heif_context_free(ctx)
    return out


def split_nals(sample):
    """[uint32 BE length][NAL]... -> [NAL bytes]."""
    out, pos = [], 0
    while pos + 4 <= len(sample):
        n = struct.unpack(">I", sample[pos:pos + 4])[0]
        out.append(sample[pos + 4:pos + 4 + n])
        pos += 4 + n
    return out


def slice_nals(au):
    """The VCL NALs (types 0..31) of a length-prefixed access unit or sample."""
    return [n for n in split_nals(au) if ((n[0] >> 1) & 0x3F) < 32]


def _boxes(buf, start, end):
    pos = start
    while pos + 8 <= end:
        size, typ = struct.unpack(">I4s", buf[pos:pos + 8])
        hdr = 8
        if size == 1:
            size, hdr = struct.unpack(">Q", buf[pos + 8:pos + 16])[0], 16
        elif size == 0:
            size = end - pos
        yield typ.decode(errors="replace"), pos + hdr, pos + size
        pos += size


def _stbl_children(buf):
    """Per track (in file order): {box type: (start, end)} of the children of moov/trak/mdia/minf/stbl."""
    out = []
    for typ, s, e in _boxes(buf, 0, len(buf)):
        if typ != "moov":
            continue
        for t2, s2, e2 in _boxes(buf, s, e):
            if t2 != "trak":
                continue
            found, stack = {}, [(s2, e2)]
            while stack:
                a, b = stack.pop()
                for t3, s3, e3 in _boxes(buf, a, b):
                    if t3 in ("mdia", "minf", "stbl"):
                        stack.append((s3, e3))
                    else:
                        found[t3] = (s3, e3)
            out.append(found)
    return out


def sync_samples(path):
    """Per track (in file order): None if the sample table has no 'stss' (every sample is a sync sample), else the 1-based
    sync sample numbers listed in it."""
    buf = open(path, "rb").read()
    out = []
    for found in _stbl_children(buf):
        stss = None
        if "stss" in found:
            s3 = found["stss"][0]
            n = struct.unpack(">I", buf[s3 + 4:s3 + 8])[0]
            stss = [struct.unpack(">I", buf[s3 + 8 + 4 * i:s3 + 12 + 4 * i])[0] for i in range(n)]
        out.append(stss)
    return out


def parameter_sets(path):
    """Per track (in file order): the VPS / SPS / PPS NALs of its 'hvcC' (stsd/hvc1/hvcC), length-prefixed like a sample, so
    that parameter_sets(path)[t] + sample is a decodable access unit."""
    buf = open(path, "rb").read()
    out = []
    for found in _stbl_children(buf):
        ps = b""
        if "stsd" in found:
            s, e = found["stsd"]
            for typ, s1, e1 in _boxes(buf, s + 8, e):                  # full box header + entry_count
                if typ != "hvc1":
                    continue
                for t2, s2, e2 in _boxes(buf, s1 + 78, e1):            # VisualSampleEntry fields
                    if t2 != "hvcC":
                        continue
                    pos, narr = s2 + 23, buf[s2 + 22]
                    for _ in range(narr):
                        nn = struct.unpack(">H", buf[pos + 1:pos + 3])[0]
                        pos += 3
                        for _ in range(nn):
                            ln = struct.unpack(">H", buf[pos:pos + 2])[0]
                            ps += struct.pack(">I", ln) + buf[pos + 2:pos + 2 + ln]
                            pos += 2 + ln
        out.append(ps)
    return out
