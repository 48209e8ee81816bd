"""Uniform batches of more than 65535 images through the driver kernels that put the image on grid y: resize, frame
conversion and the occlusion check launch them in chunks of at most 65535 images.  A batch of 2 x 2 images must equal, bit
for bit, the same op run on its two halves, each of which is one launch."""
import pytest
import torch

from unimatch_b200 import ops

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100
N = 65535 + 38                          # two chunks, the second one short


def _chunked(fn, *halves):
    """fn on the whole batch (two launches) and on each half (one launch each), outputs concatenated"""
    before = ops.launch_count()
    whole = fn(*[torch.cat(h) for h in halves])
    assert ops.launch_count() - before == 2
    a, b = fn(*[h[0] for h in halves]), fn(*[h[1] for h in halves])
    whole, a, b = [r if isinstance(r, (tuple, list)) else (r,) for r in (whole, a, b)]
    return whole, [torch.cat(p) for p in zip(a, b)]


def _split(x, k):
    return x[:k], x[k:]


def test_resize_bilinear_over_65535_planes():
    # Plane n = b C + c is scaled by scale[c].  The second chunk starts at plane 65535: with C = 2 that is channel 1, so a
    # kernel taking the channel from the chunk-local index would scale it by scale[0]; C = 3 covers the third scale.
    g = torch.Generator(device="cuda").manual_seed(0)
    for scale in ([0.5, -1.25], [0.5, 2.0, -1.25]):
        c = len(scale)
        b = (N + c - 1) // c
        x = torch.randn((b, c, 2, 2), device="cuda", generator=g)
        for flip in (False, True):
            whole, halves = _chunked(lambda t: _OPS.resize_bilinear(t, 3, 5, scale, flip), _split(x, b // 2))
            assert torch.equal(whole[0], halves[0])


def test_frames_to_planar_over_65535_frames():
    g = torch.Generator(device="cuda").manual_seed(1)
    frames = torch.randint(0, 256, (N, 2, 2, 3), device="cuda", dtype=torch.uint8, generator=g)
    for transpose in (False, True):
        whole, halves = _chunked(lambda f: _OPS.frames_to_planar(f, 3, 4, transpose), _split(frames, N // 2))
        assert torch.equal(whole[0], halves[0])
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    whole, halves = _chunked(lambda f: _OPS.frames_to_planar_normalized(f, 3, 4, mean, std), _split(frames, N // 2))
    assert torch.equal(whole[0], halves[0])


def test_fb_consistency_over_65535_pairs():
    g = torch.Generator(device="cuda").manual_seed(2)
    fwd = torch.randn((N, 2, 2, 2), device="cuda", generator=g)
    bwd = torch.randn((N, 2, 2, 2), device="cuda", generator=g)
    k = N // 2 + 1
    whole, halves = _chunked(lambda f, b: _OPS.fb_consistency(f, b, 0.01, 0.5), _split(fwd, k), _split(bwd, k))
    assert 0 < whole[0].sum() < whole[0].numel()                 # both outcomes occur
    for w, h in zip(whole, halves):
        assert torch.equal(w, h)
    whole, halves = _chunked(lambda f, b: _OPS.fb_consistency_error(f, b, 0.01, 0.5), _split(fwd, k), _split(bwd, k))
    for w, h in zip(whole, halves):
        assert torch.equal(w, h)
