"""Numpy statement of the leaderboard submission files (evaluate_flow.py:19-156, evaluate_stereo.py:28-298).

Each format's payload and header, the uint16 cast rule, the resize-back rescale and the geometry each reference driver uses,
written out step by step so that `um_encode_submission` can be checked against it bit for bit:

  * `.flo`  writeFlow (utils/frame_utils.py:70-99): b'PIEH', int32 w, int32 h, then (u, v) float32 little-endian, row-major;
  * KITTI flow PNG  writeFlowKITTI (:117-121): 16-bit RGB, R = q(64 u + 32768), G = q(64 v + 32768), B = 1, where
    `64.0 * uv + 2 ** 15` is evaluated in float32 (a float32 multiply, then a float32 add);
  * KITTI disparity PNG  `(disp * 256.).astype(np.uint16)` (evaluate_stereo.py:91): 16-bit grey, q(256 d) in float32;
  * `.pfm`  write_pfm (utils/file_io.py:98-127): b'Pf\\n', b'%d %d\\n' % (w, h), b'-1.000000\\n' (little-endian scale), then
    float32 little-endian rows from the bottom row up (np.flipud).

q is numpy's float -> uint16 cast as it behaves on x86-64 for float32 and float64 sources.  In C that conversion is undefined
for out-of-range values, so it is stated here rather than called: truncate toward zero to int32; NaN, +-inf and anything
whose truncation does not fit int32 become INT32_MIN; keep the low 16 bits.  So -1.5 -> 65535, -0.5 -> 0, 65536 -> 0,
70000.7 -> 4464, -70000.2 -> 61072, 1e10 -> 0, NaN -> 0.

The PNG payload is the filtered scanlines: row 0 with filter byte 0, every other row with the "Up" filter (filter byte 2,
each byte minus the byte above it, mod 256).  `decode_png` reads any 8- or 16-bit greyscale / RGB PNG with the stdlib.
"""
import struct
import zlib

import numpy as np

FLO, KITTI_FLOW_PNG, KITTI_DISP_PNG, PFM = 0, 1, 2, 3
TAG = b"PIEH"                      # np.array([202021.25], np.float32).tobytes()

_f32 = np.float32


def numpy_u16(x):
    """numpy's x86-64 float -> uint16 cast of a float32 / float64 array, stated explicitly."""
    x = np.asarray(x, dtype=np.float64)               # exact for float32 sources
    fits = (x >= -2147483648.0) & (x < 2147483648.0)  # trunc(x) fits int32 (NaN compares false)
    t = np.where(fits, np.trunc(np.where(fits, x, 0.0)), -2147483648.0).astype(np.int64)
    return (t & 0xFFFF).astype(np.uint16)


def fma32(a, b, c):
    """Correctly rounded float32 fma(a, b, c) of float32 arrays: a * b is exact in float64, the float64 sum is rounded to
    odd (sticky last bit, from its exact error) so that the final rounding to float32 is the single correct one."""
    a, b, c = (np.asarray(v, dtype=np.float64) for v in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        return _fma32(a, b, c)


def _fma32(a, b, c):
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                   # TwoSum: s + err == p + c exactly (finite values)
    bits = s.view(np.uint64)
    inexact = np.isfinite(s) & (err != 0) & ((bits & 1) == 0)
    toward = np.where(err > 0, np.inf, -np.inf)
    s = np.where(inexact, np.nextafter(s, toward), s)
    return s.astype(np.float32)


def _mul(a, b):
    with np.errstate(invalid="ignore", over="ignore"):
        return (np.asarray(a, np.float32) * np.asarray(b, np.float32)).astype(np.float32)


def bilinear_align_corners(x, ho, wo):
    """x: float32 [C, hi, wi] -> [C, ho, wo], the arithmetic of `um_resize_bilinear` (ATen's align-corners bilinear): fp32
    source coordinates, truncated indices, lambda weights, and the blend's two fmas and one fma as the kernel rounds them."""
    x = np.asarray(x, dtype=np.float32)
    _, hi, wi = x.shape
    sy = _f32(_f32(hi - 1) / _f32(ho - 1)) if ho > 1 else _f32(0)
    sx = _f32(_f32(wi - 1) / _f32(wo - 1)) if wo > 1 else _f32(0)
    fy = _mul(sy, np.arange(ho, dtype=np.float32))
    fx = _mul(sx, np.arange(wo, dtype=np.float32))
    y0, x0 = fy.astype(np.int64), fx.astype(np.int64)
    y1, x1 = y0 + (y0 < hi - 1), x0 + (x0 < wi - 1)
    ly, lx = (fy - y0.astype(np.float32)).astype(np.float32), (fx - x0.astype(np.float32)).astype(np.float32)
    hy, hx = (_f32(1) - ly).astype(np.float32), (_f32(1) - lx).astype(np.float32)
    ly, hy = ly[:, None], hy[:, None]
    v00, v01 = x[:, y0][:, :, x0], x[:, y0][:, :, x1]
    v10, v11 = x[:, y1][:, :, x0], x[:, y1][:, :, x1]
    row0 = fma32(lx, v01, _mul(hx, v00))
    row1 = fma32(hx, v10, _mul(lx, v11))
    return np.ascontiguousarray(fma32(hy, row0, _mul(ly, row1)))


def rescale_back(v, ori, inf):
    """The reference's rescale after the resize back: (x * ori) / inf, two float32 roundings (evaluate_flow.py:67-70,
    evaluate_stereo.py:87), not x * (ori / inf)."""
    with np.errstate(over="ignore", invalid="ignore"):
        return ((np.asarray(v, np.float32) * _f32(ori)).astype(np.float32) / _f32(inf)).astype(np.float32)


CANONICAL_NAN = np.uint32(0x7FFFFFFF)


def device_nans(x):
    """NaNs as a CUDA device returns them from arithmetic: every floating-point operation there gives the canonical NaN
    0x7fffffff, whatever NaN went in (x86 keeps the input's payload, or gives 0xffc00000 for 0 * inf).  The reference's
    resize back and rescale run on the GPU, so their NaNs are canonical too."""
    x = np.array(x, dtype=np.float32)
    x.view(np.uint32)[np.isnan(x)] = CANONICAL_NAN
    return x


def resize_back(pred, ori):
    """pred: float32 [C, h, w] at the inference size -> [C, *ori]: the resize, then u (and disparity) rescaled by the widths,
    v by the heights; every NaN of the result canonical (`device_nans`)."""
    pred = np.asarray(pred, dtype=np.float32)
    _, h, w = pred.shape
    r = bilinear_align_corners(pred, ori[0], ori[1])
    out = np.empty_like(r)
    out[0] = rescale_back(r[0], ori[1], w)
    if r.shape[0] > 1:
        out[1] = rescale_back(r[1], ori[0], h)
    return device_nans(out)


def crop(pred, top, left, h, w):
    return np.ascontiguousarray(np.asarray(pred, dtype=np.float32)[:, top:top + h, left:left + w])


def padding(ori, padding_factor, mode):
    """InputPadder (utils/utils.py:6-24): (top, left, padded size) -- centred for mode 'sintel', bottom-only in height else."""
    ph, pw = (-ori[0]) % padding_factor, (-ori[1]) % padding_factor
    top = ph // 2 if mode == "sintel" else 0
    return top, pw // 2, (ori[0] + ph, ori[1] + pw)


def nearest_size(ori, padding_factor):
    return (int(np.ceil(ori[0] / padding_factor)) * padding_factor, int(np.ceil(ori[1] / padding_factor)) * padding_factor)


def geometry(task, protocol, ori, padding_factor, inference_size=None):
    """How the reference driver of (task, protocol) brings an (H, W) sample to the model and back:
    ('pad', top, left, padded size) -- InputPadder, then its unpad crop -- or ('resize', inference size) -- resize to it and
    back with the rescale, even when it equals the original size (the rescale can still round) -- or ('none',) -- the
    model sees the sample as it is (ETH3D when the nearest multiple is the original size)."""
    ori = (int(ori[0]), int(ori[1]))
    if task == "stereo" and protocol == "eth3d":
        size = nearest_size(ori, padding_factor) if inference_size is None else tuple(int(s) for s in inference_size)
        return ("none",) if size == ori else ("resize", size)
    if inference_size is not None:
        return ("resize", (int(inference_size[0]), int(inference_size[1])))
    mode = "kitti" if (task, protocol) == ("flow", "kitti") else "sintel"
    top, left, size = padding(ori, padding_factor, mode)
    return ("pad", top, left, size)


def to_original(pred, geom, ori):
    """The model's output [C, h, w] -> [C, *ori] under `geometry(...)`."""
    if geom[0] == "resize":
        return resize_back(pred, ori)
    top, left = (geom[1], geom[2]) if geom[0] == "pad" else (0, 0)
    return crop(pred, top, left, ori[0], ori[1])


# ---- payloads (the bytes after the header) --------------------------------------------------------------------------------
def flo_payload(flow):
    """flow [2, H, W] float32: writeFlow's float64 interleave, then astype(float32)."""
    _, h, w = flow.shape
    tmp = np.zeros((h, w * 2))
    tmp[:, np.arange(w) * 2] = flow[0]
    tmp[:, np.arange(w) * 2 + 1] = flow[1]
    return tmp.astype("<f4").tobytes()


def kitti_flow_pixels(flow):
    """flow [2, H, W] float32 -> uint16 [H, W, 3] as the file holds it (R = u', G = v', B = 1)."""
    with np.errstate(over="ignore", invalid="ignore"):
        uv = (np.moveaxis(np.asarray(flow, np.float32), 0, -1) * _f32(64)).astype(np.float32)
        uv = (uv + _f32(32768)).astype(np.float32)
    px = np.empty(uv.shape[:2] + (3,), dtype=np.uint16)
    px[..., :2] = numpy_u16(uv)
    px[..., 2] = 1
    return px


def kitti_disp_pixels(disp):
    """disp [H, W] float32 -> uint16 [H, W]"""
    with np.errstate(over="ignore", invalid="ignore"):
        return numpy_u16((np.asarray(disp, np.float32) * _f32(256)).astype(np.float32))


def png_scanlines(pixels):
    """uint8 or uint16 [H, W(, channels)] -> the filtered scanlines (big-endian samples): row 0 unfiltered, the others "Up"."""
    px = np.asarray(pixels)
    h = px.shape[0]
    raw = np.ascontiguousarray(px.astype(">u2" if px.dtype == np.uint16 else np.uint8)).view(np.uint8).reshape(h, -1)
    filt = raw.copy()
    filt[1:] = raw[1:] - raw[:-1]                     # uint8 arithmetic wraps mod 256
    kind = np.full((h, 1), 2, dtype=np.uint8)
    kind[0] = 0
    return np.concatenate([kind, filt], axis=1).tobytes()


def pfm_payload(disp):
    return np.ascontiguousarray(np.flipud(np.asarray(disp, np.float32))).astype("<f4").tobytes()


def payload(values, fmt):
    """values: [C, H, W] float32 at the original size -> the payload bytes of `fmt`."""
    if fmt == FLO:
        return flo_payload(values)
    if fmt == KITTI_FLOW_PNG:
        return png_scanlines(kitti_flow_pixels(values))
    if fmt == KITTI_DISP_PNG:
        return png_scanlines(kitti_disp_pixels(values[0]))
    if fmt == PFM:
        return pfm_payload(values[0])
    raise ValueError("unknown format %r" % (fmt,))


# ---- headers -------------------------------------------------------------------------------------------------------------
def flo_header(h, w):
    return TAG + np.array(w).astype(np.int32).tobytes() + np.array(h).astype(np.int32).tobytes()


def pfm_header(h, w):
    return b"Pf\n" + b"%d %d\n" % (w, h) + b"%f\n" % -1


# ---- PNG reading (stdlib) ------------------------------------------------------------------------------------------------
def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def decode_png(data):
    """Non-interlaced 8- / 16-bit greyscale, RGB or RGBA PNG bytes -> numpy [H, W] or [H, W, C] (uint8 / uint16)."""
    if data[:8] != b"\x89PNG\r\n\x1a\n":
        raise ValueError("not a PNG")
    pos, idat, hdr = 8, [], None
    while pos < len(data):
        n, kind = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        if struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] != zlib.crc32(kind + body):
            raise ValueError("bad CRC in %r" % kind)
        if kind == b"IHDR":
            hdr = struct.unpack(">IIBBBBB", body)
        elif kind == b"IDAT":
            idat.append(body)
        elif kind == b"IEND":
            break
        pos += 12 + n
    w, h, depth, ctype, _, _, interlace = hdr
    if interlace or depth not in (8, 16) or ctype not in (0, 2, 6):
        raise ValueError("unsupported PNG (depth %d, colour type %d, interlace %d)" % (depth, ctype, interlace))
    ch = {0: 1, 2: 3, 6: 4}[ctype]
    bpp = ch * depth // 8
    stride = w * bpp
    raw = zlib.decompress(b"".join(idat))
    out = np.zeros((h, stride), dtype=np.uint8)
    prev = np.zeros(stride, dtype=np.int64)
    for y in range(h):
        f = raw[y * (stride + 1)]
        line = np.frombuffer(raw, np.uint8, stride, y * (stride + 1) + 1).astype(np.int64)
        if f == 0:
            cur = line
        elif f == 2:
            cur = (line + prev) & 0xFF
        elif f in (1, 3, 4):
            cur = np.zeros(stride, dtype=np.int64)
            for i in range(stride):
                a = cur[i - bpp] if i >= bpp else 0
                c = prev[i - bpp] if i >= bpp else 0
                pred = a if f == 1 else ((a + prev[i]) >> 1 if f == 3 else _paeth(a, prev[i], c))
                cur[i] = (line[i] + pred) & 0xFF
        else:
            raise ValueError("bad filter type %d" % f)
        out[y] = cur
        prev = cur
    px = out.view(">u2").astype(np.uint16) if depth == 16 else out
    return px.reshape(h, w, ch) if ch > 1 else px.reshape(h, w)
