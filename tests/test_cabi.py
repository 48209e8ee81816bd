"""The C-ABI shared library loads without a GPU and exports every symbol include/unimatch_sm100.h declares."""
import ctypes
import os
import re

from unimatch_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "unimatch_sm100.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(um_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported():
    lib = ctypes.CDLL(ops.LIB_PATH)
    names = _declared()
    assert len(names) >= 17
    for n in names:
        assert hasattr(lib, n), "missing export: " + n
    assert sorted(ops.SYMBOLS) == names


def test_abi_version_matches_header_and_build_info():
    text = open(os.path.join(ROOT, "include", "unimatch_sm100.h")).read()
    declared = int(re.search(r"#define UM_ABI_VERSION (\d+)", text).group(1))
    assert declared == 4
    assert ops.LIB.um_abi_version() == declared
    info = ops.build_info()
    assert "sm_90a" in info
    assert "abi=%d " % declared in info


def test_bad_arguments_are_reported_without_a_gpu():
    # argument validation happens before any CUDA call, so it can run here
    rc = ops.LIB.um_flow_warp(None, None, None, 1, 4, 4, 2, None)
    assert rc == -22
    assert b"um_flow_warp" in ops.LIB.um_last_error()
    g = ops.AttnGeom(10, 10, 3, 2, 0, 0, 0)      # 10 not divisible by 3
    one = ctypes.c_void_p(16)
    rc = ops.LIB.um_window_attention(one, one, one, one, 2, 0, 128, 128, 128, 128, ctypes.byref(g), None, 0, 0, None)
    assert rc == -22


def _conv_desc(**kw):
    d = ops.ConvDesc()
    one = 1024                                     # any non-null, 16-byte aligned address: validation never dereferences it
    d.src[0] = one; d.cin_p[0] = 128; d.nsrc = 1
    d.batch, d.h, d.w = 1, 16, 16
    d.weights = one
    d.kh = d.kw = 1
    d.cout = d.cout_p = d.bn = 128
    d.mode, d.act = ops.CONV_LINEAR, ops.ACT_NONE
    d.out_f32 = one; d.ld_f32 = 128
    d.stride = 1
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_conv_descriptor_validation_without_a_gpu():
    """um_conv2d_tc rejects malformed descriptors with -EINVAL and a message before touching the device."""
    bad = [
        dict(bn=32),                                               # tile widths are 16, 64, 96, 128, 192, 256
        dict(cout_p=130),                                          # cout_p must be a multiple of bn
        dict(stride=3),
        dict(kh=8, kw=8),                                          # more than 49 taps
        dict(mode=ops.CONV_GRU_ZR),                                # needs cout 256, h, both outputs
        dict(mode=ops.CONV_LN),                                    # needs gamma / beta
        dict(out_f32=None),                                        # no output at all
    ]
    for kw in bad:
        rc = ops.LIB.um_conv2d_tc(ctypes.byref(_conv_desc(**kw)), None)
        assert rc == -22, kw
        assert b"um_conv2d_tc" in ops.LIB.um_last_error(), kw
    d = _conv_desc()
    d.cin_p[0] = 100                                               # padded channels must be multiples of 64
    assert ops.LIB.um_conv2d_tc(ctypes.byref(d), None) == -22


def test_ffn_descriptor_validation_without_a_gpu():
    """um_ffn_tc rejects malformed descriptors with -EINVAL before touching the device."""
    def desc(**kw):
        d = ops.FfnDesc()
        one = 1024
        d.src[0] = d.src[1] = one
        d.rows, d.src_plane_stride = 512, 512 * 128
        d.w1 = d.w2 = one
        d.hidden = 1024
        d.gamma = d.beta = one
        d.out_f32, d.ld_f32 = one, 128
        for k, v in kw.items():
            setattr(d, k, v)
        return d
    for kw in (dict(rows=384), dict(rows=0), dict(hidden=1000), dict(out_f32=None), dict(src_plane_stride=100),
               dict(gamma=None), dict(ld_f32=130), dict(residual=1028, ld_res=128)):
        assert ops.LIB.um_ffn_tc(ctypes.byref(desc(**kw)), None) == -22, kw
        assert b"um_ffn_tc" in ops.LIB.um_last_error(), kw
    assert not ops.ffn_tc_supported(384) and ops.ffn_tc_supported(512)


def test_conv7x7_validation_without_a_gpu():
    one = ctypes.c_void_p(1024)
    args = dict(cin=3, stride=2, cout=64)
    for change in (dict(cin=4), dict(stride=3), dict(cout=24), dict(cout=256)):
        a = dict(args, **change)
        rc = ops.LIB.um_conv7x7_small(one, one, 1, 1, 2, 32, 32, a["cin"], a["stride"], one, None, a["cout"], 0, None, None,
                                      one, 64, None, 0, None)
        assert rc == -22, change
        assert b"um_conv7x7_small" in ops.LIB.um_last_error()


def test_colouring_batches_over_65535_images_are_refused_without_a_gpu():
    """The colouring kernels put the image on grid y (at most 65535 CTAs): a larger uniform batch is refused up front."""
    one = ctypes.c_void_p(1024)
    for name in ("um_flow_to_image", "um_disparity_to_image", "um_depth_to_image"):
        rc = getattr(ops.LIB, name)(one, one, 12, 48, one, 65536, 4, 4, None)      # 4 x 4 pictures, 12-byte rows
        assert rc == -22, name
        assert name.encode() in ops.LIB.um_last_error()
