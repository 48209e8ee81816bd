"""The TSDF ray cast on the device: `TSDFVolume.render` against the float32 statement (tests/refops_render.py), depth,
colour and normal bit for bit, on fused random clips, the analytic clip volumes, uploaded analytic fields with unobserved
voxels, batches mixing cameras inside, outside and facing away from the box, an empty volume and a `DepthFusionRunner`
volume; the kernel replayed from a CUDA graph against the eager call."""
import numpy as np
import pytest
import torch

import refops_fusion as RF
import refops_mesh as RM
import refops_render as RR
from test_fusion_cpu import covering_scene
from test_fusion_gpu import DIMS, K, ORIGIN, VS, _clip, _model, _planes, _random_clip, _runner_volume
from test_mesh_gpu import _upload
from unimatch_b200.fusion import TSDFVolume, fuse_depths
from unimatch_b200.inference import DepthFusionRunner, _camera_to_world

pytestmark = pytest.mark.gpu
_OPS = torch.ops.unimatch_sm100


def _check_render(vol, Kc, poses, h, w, near=0.0, far=None, min_hits=1):
    """render() against the float32 statement on the downloaded planes; returns the images"""
    out = vol.render(Kc, poses, (h, w), near=near, far=far)
    assert out["depth"].shape == (len(poses), h, w) and out["depth"].device == vol.device
    assert out["color"].dtype == torch.uint8 and out["normal"].shape == (len(poses), h, w, 3)
    Kf = np.asarray(Kc, np.float32)
    rd, rc, rn = RR.raycast(_planes(vol), vol.origin, vol.voxel_size, vol.trunc, _camera_to_world(poses), Kf, h, w,
                            np.float32(near), np.inf if far is None else np.float32(far), np.float32)
    assert np.array_equal(out["depth"].cpu().numpy().view(np.uint32), rd.view(np.uint32))
    assert np.array_equal(out["color"].cpu().numpy(), rc)
    assert np.array_equal(out["normal"].cpu().numpy().view(np.uint32), rn.view(np.uint32))
    assert (rd > 0).sum() >= min_hits
    return out


@pytest.mark.parametrize("seed", [1, 3])
def test_fused_random_clip(seed):
    d, frames, poses = _random_clip(6, 40, 56, seed=seed)
    vol = TSDFVolume(ORIGIN, VS, DIMS, device="cuda")
    fuse_depths(vol, torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda(), K, poses)
    out = _check_render(vol, K, poses, 40, 56, min_hits=1000)
    again = vol.render(K, poses, (40, 56))
    assert all(torch.equal(out[k], again[k]) for k in out)
    _check_render(vol, K, poses[:2], 40, 56, near=2.0, far=3.5, min_hits=100)


@pytest.mark.parametrize("clip", ["constant_plane", "tilted_plane", "sphere"])
def test_analytic_clip_volumes(clip):
    scene, Kc, poses = getattr(RF, clip + "_clip")()
    h, w = (24, 32) if clip == "constant_plane" else (48, 64)
    vs = 1 / 32 if clip == "constant_plane" else 0.01
    origin, dims = ((-0.3125, -0.3125, 0.875), (20, 20, 8)) if clip == "constant_plane" else covering_scene(scene)
    depths = np.stack([RF.render(scene, Kc, P, h, w) for P in poses]).astype(np.float32)
    frames = np.random.default_rng(5).integers(0, 256, (len(poses), h, w, 3), dtype=np.uint8)
    vol = TSDFVolume(origin, vs, dims, device="cuda")
    Kf = np.array(Kc, np.float32)
    p32 = [p.astype(np.float32) for p in poses]
    fuse_depths(vol, torch.from_numpy(depths).cuda(), torch.from_numpy(frames).cuda(), Kf, p32)
    _check_render(vol, Kf, p32, h, w, min_hits=100)


@pytest.mark.parametrize("name,field", [
    ("sphere", RM.sphere((0.013, -0.021, 0.017), 0.61)),
    ("torus", RM.torus((0.011, -0.013, 0.007), 0.55, 0.21)),
])
def test_uploaded_fields_with_unobserved_voxels(name, field):
    vs = 1 / 32
    origin, dims = (-1.0, -1.0, -0.75), (64, 61, 47)
    planes = RM.sdf_volume(field, origin, vs, dims, 4 * vs)
    g = np.random.default_rng(11)
    planes["weight"] = planes["weight"] * (g.random(planes["weight"].shape) > 0.02)
    planes["color"] = g.uniform(0, 255, planes["color"].shape)
    vol = _upload(TSDFVolume(origin, vs, dims, trunc=4 * vs, device="cuda"), planes)
    Kc = np.array([[60.0, 0, 40.0], [0, 60.0, 30.0], [0, 0, 1]], np.float32)
    poses = [RF.pose(RF.rot("y", a) @ RF.rot("x", 0.3), RF.rot("y", a) @ RF.rot("x", 0.3) @ [0.0, 0.0, -2.2]).astype(np.float32)
             for a in (0.0, 1.3, 2.9)]
    _check_render(vol, Kc, poses, 60, 80, min_hits=2000)


def test_cameras_inside_outside_and_facing_away():
    d, frames, poses = _random_clip(6, 40, 56, seed=2)
    vol = TSDFVolume(ORIGIN, VS, DIMS, device="cuda")
    fuse_depths(vol, torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda(), K, poses)
    centre = np.array(ORIGIN) + np.array(DIMS) * VS / 2
    mixed = [poses[0],                                                        # outside, facing the box
             RF.pose(np.eye(3), centre).astype(np.float32),                   # inside
             RF.pose(RF.rot("y", 2.0), centre + [0.3, 0.2, -0.4]).astype(np.float32),
             RF.pose(RF.rot("x", np.pi), [0.0, 0.0, -1.0]).astype(np.float32),  # outside, facing away
             RF.pose(np.eye(3), [50.0, 0.0, 0.0]).astype(np.float32)]         # beside the box
    out = _check_render(vol, K, mixed, 40, 56, min_hits=100)
    assert not out["depth"][3:].any() and not out["color"][3:].any() and not out["normal"][3:].any()


def test_empty_volume_and_no_cameras():
    vol = TSDFVolume(ORIGIN, VS, DIMS, device="cuda")
    out = _check_render(vol, K, [np.eye(4, dtype=np.float32)], 40, 56, min_hits=0)
    assert not out["depth"].any() and not out["color"].any() and not out["normal"].any()
    none = vol.render(K, [], (40, 56))
    assert none["depth"].shape == (0, 40, 56) and none["color"].shape == (0, 40, 56, 3) and none["normal"].shape == (0, 40, 56, 3)


def test_raycast_replayed_from_a_cuda_graph_equals_render():
    d, frames, poses = _random_clip(4, 40, 56, seed=4)
    vol = TSDFVolume(ORIGIN, VS, DIMS, device="cuda")
    fuse_depths(vol, torch.from_numpy(d).cuda(), torch.from_numpy(frames).cuda(), K, poses)
    c2w = torch.from_numpy(_camera_to_world(poses[:2])).cuda()
    args = (vol.tsdf, vol.weight, vol.color, vol.origin, vol.voxel_size, vol.trunc)
    intr = (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), 0.0, float("inf"))
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        _OPS.tsdf_raycast(*args, c2w, 40, 56, *intr)                         # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = _OPS.tsdf_raycast(*args, c2w, 40, 56, *intr)
    for pair in (poses[2:], poses[:2]):
        c2w.copy_(torch.from_numpy(_camera_to_world(pair)))
        graph.replay()
        ref = vol.render(K, pair, (40, 56))
        assert torch.equal(static[0], ref["depth"]) and torch.equal(static[1], ref["color"])
        assert torch.equal(static[2], ref["normal"])
        assert (ref["depth"] > 0).sum() > 100


def test_runner_volume_at_its_input_poses():
    m, kw = _model()
    frames, Kc, poses, items = _clip()
    vol = _runner_volume(Kc, poses, 64, 96)
    runner = DepthFusionRunner(m, (64, 96), 3, "cuda", Kc, vol, return_depth=False, **kw)
    list(runner.run(items))
    _check_render(runner.volume, Kc.numpy() if torch.is_tensor(Kc) else Kc, list(poses.numpy()), 64, 96, min_hits=100)
