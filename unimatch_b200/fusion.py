"""TSDF fusion of posed depth maps on the device: a dense truncated-signed-distance volume (`TSDFVolume`), the integration of
device depths and frames into it (`fuse_depths`, one `um_tsdf_integrate` launch), the zero-crossing points of its surface
with their colours (`TSDFVolume.extract_points`), its marching-cubes mesh with per-vertex normals
(`TSDFVolume.extract_mesh`), its ray-cast depth, colour and normal images from any camera (`TSDFVolume.render`, one
`um_tsdf_raycast` launch), the tracking of cameras against it (`TSDFVolume.track`, point-to-plane ICP in the um_icp_*
launches), a binary PLY writer and reader for the points and meshes (`write_ply`, `read_ply`), and exact nearest
neighbours and voxel down-sampling of point clouds (`nearest_neighbors`, `voxel_down_sample`, the um_cloud_* launches)
that `evaluation.reconstruction_metrics` scores reconstructions with, the rasterisation of triangle meshes from any camera
into depth, face and colour images (`render_mesh`, the um_mesh_* launches) and the visibility of points in depth maps
(`visible_points`, one `um_visible_points` launch), which culls both sets to what the cameras saw before scoring, and the
multi-view geometric consistency filter of depth maps (`filter_depths` over a `sequence_sources` table, one
`um_depth_consistency` launch) with the export of valid depths as coloured world points (`depth_points`).  The kernels'
arithmetic is stated in include/unimatch_sm100.h; `DepthFusionRunner` (inference.py) fuses the depths of `DepthSequenceRunner` inside
each step's CUDA graph."""
import math

import numpy as np
import torch

from .inference import _OPS, _camera_to_world, _intrinsics33, _pose44, _world_to_camera
from .ops import ICP_STATE, ICP_TERMS, icp_blocks

MAX_VOXELS = 2 ** 31 - 1
MAX_MESH_INDEX = 2 ** 31 - 1                           # int32 face indices: at most this many vertices and faces


def _f32(v):
    """A Python float that is exactly the float32 the kernels receive"""
    return float(np.float32(v))


class TSDFVolume:
    """A dense TSDF volume of dims = (X, Y, Z) voxels of `voxel_size` metres (x fastest), whose low corner is `origin`: voxel
    (i, j, k) is centred at origin + (idx + 0.5) * voxel_size per axis.  Device planes, zeroed (empty): `tsdf` and `weight`
    fp32 [Z, Y, X] and `color` fp32 [3, Z, Y, X] (RGB in 0..255), 20 bytes per voxel.  `trunc` (metres, default 4 voxel
    sizes) is the truncation distance: the stored value is min(1, sdf / trunc), and a voxel more than `trunc` behind the
    observed surface is not updated.  At most 2^31 - 1 voxels."""

    def __init__(self, origin, voxel_size, dims, trunc=None, device="cuda"):
        dims = tuple(int(d) for d in dims)
        if len(dims) != 3 or min(dims) < 1:
            raise ValueError("TSDFVolume: dims must be three positive voxel counts (X, Y, Z)")
        if math.prod(dims) > MAX_VOXELS:
            raise ValueError("TSDFVolume: %d x %d x %d voxels is more than 2^31 - 1" % dims)
        if not (math.isfinite(voxel_size) and voxel_size > 0):
            raise ValueError("TSDFVolume: voxel_size must be positive and finite")
        trunc = 4.0 * _f32(voxel_size) if trunc is None else trunc
        if not (math.isfinite(trunc) and trunc > 0):
            raise ValueError("TSDFVolume: trunc must be positive and finite")
        origin = [float(o) for o in origin]
        if len(origin) != 3 or not all(math.isfinite(o) for o in origin):
            raise ValueError("TSDFVolume: origin must be three finite coordinates")
        self.origin = [_f32(o) for o in origin]
        self.voxel_size, self.trunc, self.dims = _f32(voxel_size), _f32(trunc), dims
        if torch.device(device).type != "cuda":
            raise ValueError("TSDFVolume: the volume lives on a CUDA device")
        X, Y, Z = dims
        self.tsdf = torch.zeros((Z, Y, X), dtype=torch.float32, device=device)
        self.weight = torch.zeros((Z, Y, X), dtype=torch.float32, device=device)
        self.color = torch.zeros((3, Z, Y, X), dtype=torch.float32, device=device)
        self.device = self.tsdf.device                   # with its index, as tensors on it report it

    @classmethod
    def covering(cls, intrinsics, poses, frame_size, max_depth, voxel_size, trunc=None, device="cuda"):
        """The volume over the axis-aligned box of the cameras' view frusta from depth 0 to `max_depth`, padded by `trunc`
        (default 4 voxel sizes) on every side: intrinsics [3,3] at `frame_size` = (H, W), host camera-to-world poses
        [N,4,4] (see `covering_box`)."""
        origin, dims, trunc = covering_box(intrinsics, poses, frame_size, max_depth, voxel_size, trunc)
        return cls(origin, voxel_size, dims, trunc=trunc, device=device)

    def reset(self):
        """Empty the volume (every plane zeroed)"""
        self.tsdf.zero_(), self.weight.zero_(), self.color.zero_()

    def extract_points(self):
        """The zero-crossing vertices of marching cubes on the observed voxels: points fp32 [P,3] (world coordinates) and
        their colours uint8 [P,3], on the device, ordered by voxel index, then edge axis x, y, z.  One count pass, one scan,
        one read of the count P by the host, one write pass; the result is the same from run to run."""
        with torch.cuda.device(self.device):
            offsets = _OPS.tsdf_surface_count(self.tsdf, self.weight)
            n = int(offsets[-1].item())
            return _OPS.tsdf_surface_points(self.tsdf, self.weight, self.color, self.origin, self.voxel_size, offsets, n)

    def extract_mesh(self):
        """Marching cubes on the observed voxels, on the device: points fp32 [P,3] and colors uint8 [P,3], which are
        `extract_points()`'s bit for bit and in its order; normals fp32 [P,3], unit vectors along the TSDF gradient
        (towards free space; (0, 0, 0) where the gradient vanishes); faces int32 [T,3] indices into the points,
        counter-clockwise seen from free space, ordered by cube.  A cube (the 8 voxels from (i, j, k) to (i+1, j+1, k+1))
        has faces only when all 8 of its voxels are observed, so a point whose cubes all touch an unobserved voxel is in
        no face, and a volume with a dimension below 2 has none.  Count passes for points and faces, one host read of both
        totals, then a vertex pass and a face pass; no atomics, the same result from run to run.  More than 2^31 - 1 points
        or faces is refused before the outputs are allocated."""
        with torch.cuda.device(self.device):
            point_offsets = _OPS.tsdf_surface_count(self.tsdf, self.weight)
            face_offsets = _OPS.tsdf_mesh_count(self.tsdf, self.weight)
            n_points, n_faces = torch.stack((point_offsets[-1], face_offsets[-1])).tolist()
            if max(n_points, n_faces) > MAX_MESH_INDEX:
                raise ValueError("TSDFVolume.extract_mesh: %d points and %d faces; int32 faces hold at most 2^31 - 1 of "
                                 "each" % (n_points, n_faces))
            return _OPS.tsdf_mesh(self.tsdf, self.weight, self.color, self.origin, self.voxel_size, point_offsets, n_points,
                                  face_offsets, n_faces)

    @torch.no_grad()
    def render(self, intrinsics, poses, frame_size, near=0.0, far=None):
        """The fused surface seen by N pinhole cameras, ray-cast on the device in one `um_tsdf_raycast` launch: intrinsics
        [3,3] at `frame_size` = (H, W), host camera-to-world poses [N,4,4] (as `fuse_depths` takes them).  Each pixel's ray
        through its centre is marched over the box of voxel centres between camera z-depths `near` and `far` (None: the
        box alone limits it) and ends at the first zero crossing of the trilinear TSDF from positive to negative between two
        observed samples.  Returns {'depth': fp32 [N,H,W] camera z-depth, 'color': uint8 [N,H,W,3] RGB, 'normal': fp32
        [N,H,W,3] unit world-space normals towards free space}, on the volume's device, all 0 where a ray finds no surface
        (a depth of 0 is "no estimate" to `fuse_depths` and `depth_to_image`).  A ray that first crosses from negative to
        positive (a camera inside a surface) misses.  No atomics and no host synchronisation after the one upload of the
        poses; the same result from run to run."""
        K = _intrinsics33(intrinsics, "TSDFVolume.render")
        fx, fy, cx, cy = _camera(K, "TSDFVolume.render")
        ps = [_pose44(p, "TSDFVolume.render") for p in poses]
        if not all(np.isfinite(p).all() for p in ps):
            raise ValueError("TSDFVolume.render: camera poses must be finite")
        h, w = (int(v) for v in frame_size)
        if h < 1 or w < 1 or h * w > MAX_VOXELS:
            raise ValueError("TSDFVolume.render: frame_size must be (H, W) with at most 2^31 - 1 pixels")
        if len(ps) > 65535:
            raise ValueError("TSDFVolume.render: at most 65535 cameras per call")
        near, far = _f32(near), math.inf if far is None else _f32(far)
        if not (math.isfinite(near) and near >= 0 and far > near):
            raise ValueError("TSDFVolume.render: near must be finite and >= 0, far None or greater than near")
        if not ps:
            return {"depth": torch.zeros((0, h, w), dtype=torch.float32, device=self.device),
                    "color": torch.zeros((0, h, w, 3), dtype=torch.uint8, device=self.device),
                    "normal": torch.zeros((0, h, w, 3), dtype=torch.float32, device=self.device)}
        with torch.cuda.device(self.device):
            c2w = torch.from_numpy(_camera_to_world(ps)).to(self.device)
            depth, color, normal = _OPS.tsdf_raycast(self.tsdf, self.weight, self.color, self.origin, self.voxel_size,
                                                     self.trunc, c2w, h, w, fx, fy, cx, cy, near, far)
        return {"depth": depth, "color": color, "normal": normal}

    @torch.no_grad()
    def track(self, depths, intrinsics, poses, *, levels=3, iterations=(4, 5, 10), max_distance=0.1, max_angle=20.0,
              min_inlier_fraction=0.3):
        """Track N cameras against the fused surface: frame-to-model point-to-plane ICP (KinectFusion) on the device.
        depths: device fp32 [N,H,W] (metric z-depth; zero, negative and non-finite depths are invalid), intrinsics [3,3]
        at (H, W), host camera-to-world initial poses [N,4,4] (as `fuse_depths` takes them).  Each frame is tracked on
        its own, coarse to fine over a `levels`-level depth pyramid with `iterations[i]` Gauss-Newton steps on level
        levels - 1 - i, against the volume ray-cast (`render`) at its initial pose; a pixel pairs with the model pixel
        its point projects to when they are within `max_distance` metres and their normals within `max_angle` degrees.
        A frame is tracked when no finest-level step was degenerate and at least `min_inlier_fraction` of its valid
        pixels are inliers at the end; a frame that is not tracked gets its initial pose back unchanged.  The
        arithmetic is stated in include/unimatch_sm100.h (um_icp_*).  One upload, a fixed launch sequence and one
        download.  Returns {'pose': float32 [N,4,4] camera-to-world, 'tracked': bool [N], 'inliers': int64 [N],
        'rmse': float32 [N] (the inliers' point-to-plane residual, metres)} on the host."""
        name = "TSDFVolume.track"
        if not (torch.is_tensor(depths) and depths.is_cuda and depths.dtype == torch.float32 and depths.dim() == 3):
            raise ValueError("%s: depths must be a device float32 tensor [N,H,W]" % name)
        if depths.device != self.device:
            raise ValueError("%s: depths must be on the volume's device" % name)
        n, h, w = depths.shape
        K = _intrinsics33(intrinsics, name)
        ps = [_pose44(p, name) for p in poses]
        if len(ps) != n:
            raise ValueError("%s: %d depth maps need %d poses, got %d" % (name, n, n, len(ps)))
        if not all(np.isfinite(p).all() for p in ps):
            raise ValueError("%s: camera poses must be finite" % name)
        if n > 65535:
            raise ValueError("%s: at most 65535 frames per call" % name)
        icp = _ICP(self, K, n, h, w, levels, iterations, max_distance, max_angle, min_inlier_fraction, name)
        out = {"pose": np.zeros((0, 4, 4), np.float32), "tracked": np.zeros(0, bool), "inliers": np.zeros(0, np.int64),
               "rmse": np.zeros(0, np.float32)}
        if n == 0:
            return {k: torch.from_numpy(v) for k, v in out.items()}
        with torch.cuda.device(self.device):
            poses64 = torch.from_numpy(np.stack(ps).astype(np.float64)).to(self.device)
            n_valid = torch.full((1,), n, dtype=torch.int32, device=self.device)
            packed = torch.empty((77 * n,), dtype=torch.uint8, device=self.device)     # one download
            views = (packed[:64 * n].view(torch.float32).view(n, 4, 4), packed[76 * n:],
                     packed[64 * n:72 * n].view(torch.int64), packed[72 * n:76 * n].view(torch.float32))
            icp.track(*icp.prepare(depths.contiguous()), poses64, n_valid, views)
            host = packed.cpu().numpy()
        return {"pose": torch.from_numpy(host[:64 * n].view(np.float32).reshape(n, 4, 4).copy()),
                "tracked": torch.from_numpy(host[76 * n:].astype(bool)),
                "inliers": torch.from_numpy(host[64 * n:72 * n].view(np.int64).copy()),
                "rmse": torch.from_numpy(host[72 * n:76 * n].view(np.float32).copy())}

    def _integrate(self, depths, frames, w2c, n_valid, K):
        """One um_tsdf_integrate launch: frames 0 .. n_valid - 1 of device depths [n,H,W] and uint8 frames [n,H,W,3] with
        their world-to-camera rows w2c [n,3,4] (device fp32) and the float32 intrinsics K [3,3] (host)."""
        _OPS.tsdf_integrate(self.tsdf, self.weight, self.color, self.origin, self.voxel_size, self.trunc, depths, frames, w2c,
                            float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), n_valid)


ICP_MIN_INLIERS = 36            # 6 x 6: at least as many inliers as the system has unknowns, times six
ICP_MIN_PIVOT = 1e-2            # smallest Cholesky pivot of the Jacobi-scaled 6 x 6 system (see tests/test_icp_cpu.py)


def icp_levels(K, h, w, levels):
    """[(fx, fy, cx, cy, h, w)] of the depth pyramid's levels, finest first: float32 intrinsics (fx/2, fy/2, (cx - 0.5)/2,
    (cy - 0.5)/2 per level, so pixel x is centred at x on every level) and floor-halved sizes."""
    f32 = np.float32
    fx, fy, cx, cy = (f32(K[0][0]), f32(K[1][1]), f32(K[0][2]), f32(K[1][2]))
    out = [(fx, fy, cx, cy, h, w)]
    for _ in range(levels - 1):
        fx, fy = f32(fx * f32(0.5)), f32(fy * f32(0.5))
        cx, cy = f32(f32(cx - f32(0.5)) * f32(0.5)), f32(f32(cy - f32(0.5)) * f32(0.5))
        h, w = h // 2, w // 2
        out.append((fx, fy, cx, cy, h, w))
    return [(float(a), float(b), float(c), float(d), hh, ww) for a, b, c, d, hh, ww in out]


class _ICP:
    """The device buffers and the fixed launch sequence of tracking n frames of h x w against `volume`
    (`TSDFVolume.track`, and `DepthFusionRunner(track=True)` one frame at a time)."""

    def __init__(self, volume, K, n, h, w, levels, iterations, max_distance, max_angle, min_inlier_fraction, name):
        if isinstance(levels, bool) or not isinstance(levels, int) or levels < 1:
            raise ValueError("%s: levels must be a positive int" % name)
        its = tuple(iterations)
        if len(its) != levels or not all(isinstance(i, int) and not isinstance(i, bool) and i >= 0 for i in its) \
                or its[-1] < 1:
            raise ValueError("%s: iterations must give levels non-negative ints, coarse to fine, at least 1 on the finest"
                             % name)
        if h >> (levels - 1) < 2 or w >> (levels - 1) < 2 or h * w > MAX_VOXELS:
            raise ValueError("%s: a %d x %d frame is too small for %d pyramid levels (2 x 2 on the coarsest)"
                             % (name, h, w, levels))
        with np.errstate(over="ignore"):
            max_distance = _f32(max_distance) if math.isfinite(max_distance) else math.nan
        if not (math.isfinite(max_distance) and max_distance > 0):                # the float32 value the kernel gets
            raise ValueError("%s: max_distance must be positive and finite in float32" % name)
        if not (math.isfinite(max_angle) and 0 < max_angle <= 180):
            raise ValueError("%s: max_angle must be in (0, 180] degrees" % name)
        if not (math.isfinite(min_inlier_fraction) and 0 <= min_inlier_fraction <= 1):
            raise ValueError("%s: min_inlier_fraction must be in [0, 1]" % name)
        _camera(K, name)
        self.volume, self.n = volume, n
        self.levels = icp_levels(K.numpy(), h, w, levels)
        self.iterations = its[::-1]                                       # per level, finest first
        self.max_distance = max_distance
        self.cos_max_angle = _f32(math.cos(math.radians(max_angle)))
        self.min_inlier_fraction = float(min_inlier_fraction)
        dev = volume.device
        if n:
            self.state = torch.zeros((n, ICP_STATE), dtype=torch.float64, device=dev)
            rows = torch.eye(4, dtype=torch.float32, device=dev)[:3].repeat(n, 1, 1)
            self.c2w, self.w2c = rows.clone(), rows.clone()                # the reference rows
            self.w2c_out = rows.clone()                                    # the tracked poses' rows
            self.partials = torch.empty((n * icp_blocks(h, w) * ICP_TERMS,), dtype=torch.float64, device=dev)

    def prepare(self, depth):
        """The pyramid of device depths [n, h, w] (contiguous fp32) and its live normals, finest first"""
        pyramid = [depth]
        for _ in self.levels[1:]:
            pyramid.append(_OPS.icp_downsample(pyramid[-1], self.volume.trunc))
        return pyramid, [_OPS.icp_normals(d, *lv[:4]) for d, lv in zip(pyramid, self.levels)]

    def track(self, pyramid, normals, poses64, n_valid, outputs, correction=None):
        """Launch the schedule for frames 0 .. n_valid - 1: fp64 initial poses [n, 4, 4] (corrected on the left by the fp64
        [4, 4] `correction` when given, which a tracked frame then updates), outputs = (pose fp32 [n, 4, 4], tracked uint8
        [n], inliers int64 [n], rmse fp32 [n]); the tracked poses' world-to-camera rows land in `w2c_out`."""
        v = self.volume
        _OPS.icp_init(poses64, correction, n_valid, self.state, self.c2w, self.w2c)
        models = [_OPS.tsdf_raycast(v.tsdf, v.weight, v.color, v.origin, v.voxel_size, v.trunc, self.c2w, lv[4], lv[5],
                                    *lv[:4], 0.0, math.inf) for lv in self.levels]

        def reduce(level):
            fx, fy, cx, cy, h, w = self.levels[level]
            _OPS.icp_reduce(pyramid[level], normals[level], models[level][0], models[level][2], self.state, self.c2w,
                            self.w2c, fx, fy, cx, cy, self.max_distance, self.cos_max_angle, n_valid, self.partials)
            return icp_blocks(h, w)

        for level in reversed(range(len(self.levels))):
            for _ in range(self.iterations[level]):
                nb = reduce(level)
                _OPS.icp_solve(self.partials, nb, n_valid, float(ICP_MIN_INLIERS), ICP_MIN_PIVOT, level == 0, self.state)
        nb = reduce(0)
        pose, tracked, inliers, rmse = outputs
        _OPS.icp_accept(self.partials, nb, n_valid, self.min_inlier_fraction, poses64 if correction is not None else None,
                        correction, self.state, pose, tracked, inliers, rmse, self.w2c_out)


def covering_box(intrinsics, poses, frame_size, max_depth, voxel_size, trunc=None):
    """(origin, dims, trunc) of `TSDFVolume.covering`: the axis-aligned box of every camera's frustum apex and the four far
    corners of its frame (pixel corners (0, 0) .. (W, H) at depth `max_depth`), in float64, padded by `trunc` on every
    side; origin is the box's low corner and dims = ceil(extent / voxel_size) per axis, so the voxels cover the box."""
    K = _intrinsics33(intrinsics, "TSDFVolume.covering").double().numpy()
    ps = [_pose44(p, "TSDFVolume.covering").astype(np.float64) for p in poses]
    if not ps:
        raise ValueError("TSDFVolume.covering: no poses")
    if not (math.isfinite(max_depth) and max_depth > 0):
        raise ValueError("TSDFVolume.covering: max_depth must be positive and finite")
    if not (math.isfinite(voxel_size) and voxel_size > 0):
        raise ValueError("TSDFVolume.covering: voxel_size must be positive and finite")
    trunc = 4.0 * _f32(voxel_size) if trunc is None else float(trunc)
    h, w = frame_size
    corners = np.array([[0.0, 0.0], [w, 0.0], [0.0, h], [w, h]])
    z = float(max_depth)
    far = np.stack([(corners[:, 0] - K[0, 2]) / K[0, 0] * z, (corners[:, 1] - K[1, 2]) / K[1, 1] * z, np.full(4, z)], 1)
    cam = np.concatenate([np.zeros((1, 3)), far], 0)                      # apex and the four far corners
    pts = np.concatenate([cam @ p[:3, :3].T + p[:3, 3] for p in ps], 0)
    lo, hi = pts.min(0) - trunc, pts.max(0) + trunc
    dims = tuple(max(1, int(math.ceil((b - a) / voxel_size))) for a, b in zip(lo, hi))
    return lo.tolist(), dims, trunc


def _check_fusion_inputs(volume, depths, frames, name):
    if not isinstance(volume, TSDFVolume):
        raise ValueError("%s: volume must be a TSDFVolume" % name)
    if not (torch.is_tensor(depths) and depths.is_cuda and depths.dtype == torch.float32 and depths.dim() == 3):
        raise ValueError("%s: depths must be a device float32 tensor [N,H,W]" % name)
    if not (torch.is_tensor(frames) and frames.is_cuda and frames.dtype == torch.uint8
            and tuple(frames.shape) == tuple(depths.shape) + (3,)):
        raise ValueError("%s: frames must be device uint8 [N,H,W,3] at the depths' size" % name)
    if depths.device != volume.device or frames.device != volume.device:
        raise ValueError("%s: depths and frames must be on the volume's device" % name)


@torch.no_grad()
def fuse_depths(volume, depths, frames, intrinsics, poses):
    """Integrate N posed depth maps into `volume` with one `um_tsdf_integrate` launch: device depths [N,H,W] (metric, as
    `infer_depth_sequence` returns them; zero, negative and non-finite depths are skipped), device uint8 frames [N,H,W,3]
    (as `infer_depth_sequence` takes them), the intrinsics [3,3] at the frames' size and the host camera-to-world poses
    [N,4,4].  Each voxel takes the frames in order and the nearest pixel of each, so fusing a sequence in one call or in
    pieces gives the same volume bit for bit.  Returns the volume."""
    _check_fusion_inputs(volume, depths, frames, "fuse_depths")
    n = depths.shape[0]
    if len(poses) != n:
        raise ValueError("fuse_depths: %d depth maps need %d poses, got %d" % (n, n, len(poses)))
    if n == 0:
        return volume
    K = _intrinsics33(intrinsics, "fuse_depths")
    w2c = _world_to_camera([_pose44(p, "fuse_depths") for p in poses])
    with torch.cuda.device(volume.device):
        w2c_dev = torch.from_numpy(w2c).to(volume.device)
        n_valid = torch.full((1,), n, dtype=torch.int32, device=volume.device)
        volume._integrate(depths.contiguous(), frames.contiguous(), w2c_dev, n_valid, K)
    return volume


def _host(t):
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def write_ply(path, points, colors, normals=None, faces=None):
    """A binary little-endian PLY of P coloured points: float x, y, z, then float nx, ny, nz when `normals` are given, and
    uchar red, green, blue per vertex; with `faces`, an element face of T triangles (property list uchar int
    vertex_indices).  `points` [P,3], `colors` [P,3] uint8, `normals` [P,3] and `faces` [T,3] (indices below P) are tensors
    (any device) or numpy arrays, as `TSDFVolume.extract_points` / `extract_mesh` return them."""
    pts = _host(points).astype("<f4", copy=False)
    col = _host(colors)
    if pts.ndim != 2 or pts.shape[1] != 3 or col.shape != pts.shape or col.dtype != np.uint8:
        raise ValueError("write_ply: expected points [P,3] and uint8 colors [P,3]")
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    props = ["float x", "float y", "float z"]
    if normals is not None:
        nrm = _host(normals).astype("<f4", copy=False)
        if nrm.shape != pts.shape:
            raise ValueError("write_ply: expected normals [P,3]")
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
        props += ["float nx", "float ny", "float nz"]
    fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    props += ["uchar red", "uchar green", "uchar blue"]
    vertex = np.empty(len(pts), dtype=fields)
    vertex["x"], vertex["y"], vertex["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
    if normals is not None:
        vertex["nx"], vertex["ny"], vertex["nz"] = nrm[:, 0], nrm[:, 1], nrm[:, 2]
    vertex["red"], vertex["green"], vertex["blue"] = col[:, 0], col[:, 1], col[:, 2]
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % len(pts)
    header += "".join("property %s\n" % p for p in props)
    body = [vertex.tobytes()]
    if faces is not None:
        tri = _host(faces)
        if tri.ndim != 2 or tri.shape[1] != 3 or tri.dtype.kind not in "iu" \
                or (tri.size and (tri.min() < 0 or tri.max() >= len(pts))):
            raise ValueError("write_ply: expected integer faces [T,3] indexing the points")
        face = np.empty(len(tri), dtype=[("n", "u1"), ("v", "<i4", 3)])
        face["n"], face["v"] = 3, tri
        header += "element face %d\nproperty list uchar int vertex_indices\n" % len(tri)
        body.append(face.tobytes())
    header += "end_header\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        for b in body:
            f.write(b)


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def read_ply(path):
    """The counterpart of `write_ply`: a binary little-endian PLY's vertices and triangles, as numpy arrays in a dict:
    'points' float32 [P,3] (x, y, z), and when present 'colors' uint8 [P,3] (red, green, blue; alpha is dropped),
    'normals' float32 [P,3] (nx, ny, nz) and 'faces' int32 [T,3].  Vertex properties may have any PLY scalar type; the
    face element holds one list property of vertex indices, every face a triangle (ScanNet's `*_vh_clean_2.ply` and
    `write_ply`'s output are both of this form).  ASCII and big-endian files, list properties elsewhere, other elements
    and faces that are not triangles are refused with ValueError."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.find(b"end_header")
    nl = data.find(b"\n", end)
    if not data.startswith(b"ply") or end < 0 or nl < 0:
        raise ValueError("read_ply: %s is not a PLY file (no 'ply' magic or no end_header)" % path)
    lines = [ln.split() for ln in data[:end].decode("ascii", "replace").splitlines()[1:]]
    elements, fmt = [], None
    for ln in lines:
        if not ln or ln[0] in ("comment", "obj_info"):
            continue
        if ln[0] == "format":
            fmt = ln[1] if len(ln) > 1 else None
        elif ln[0] == "element" and len(ln) == 3:
            elements.append((ln[1], int(ln[2]), []))
        elif ln[0] == "property" and elements:
            elements[-1][2].append(ln[1:])
        else:
            raise ValueError("read_ply: unreadable header line %r" % " ".join(ln))
    if fmt != "binary_little_endian":
        raise ValueError("read_ply: only binary_little_endian PLY is read, not %s" % fmt)
    out, offset = {}, nl + 1
    for name, count, props in elements:
        if name == "vertex":
            if any(p[0] == "list" or p[0] not in _PLY_TYPES or len(p) != 2 for p in props):
                raise ValueError("read_ply: vertex properties must be scalars of a PLY type")
            dt = np.dtype([(p[1], "<" + _PLY_TYPES[p[0]]) for p in props])
            v = np.frombuffer(data, dt, count, offset)
            offset += dt.itemsize * count
            if not all(k in dt.names for k in ("x", "y", "z")):
                raise ValueError("read_ply: the vertex element has no x, y and z")
            out["points"] = np.stack([v[k] for k in ("x", "y", "z")], 1).astype(np.float32)
            if all(k in dt.names for k in ("nx", "ny", "nz")):
                out["normals"] = np.stack([v[k] for k in ("nx", "ny", "nz")], 1).astype(np.float32)
            if all(k in dt.names for k in ("red", "green", "blue")):
                col = np.stack([v[k] for k in ("red", "green", "blue")], 1)
                if col.dtype != np.uint8:
                    raise ValueError("read_ply: colours must be uchar")
                out["colors"] = col
        elif name == "face":
            if len(props) != 1 or props[0][0] != "list" or len(props[0]) != 4 or props[0][1] not in _PLY_TYPES \
                    or props[0][2] not in _PLY_TYPES or _PLY_TYPES[props[0][2]][0] not in "iu":
                raise ValueError("read_ply: the face element must hold one list of integer vertex indices")
            dt = np.dtype([("n", "<" + _PLY_TYPES[props[0][1]]), ("v", "<" + _PLY_TYPES[props[0][2]], 3)])
            first = np.frombuffer(data, "<" + _PLY_TYPES[props[0][1]], 1, offset) if count else np.zeros(1)
            if count and first[0] != 3:
                raise ValueError("read_ply: only triangle faces are read (a face has %d vertices)" % first[0])
            f = np.frombuffer(data, dt, count, offset)       # with triangles only, the records are of one size
            if (f["n"] != 3).any():
                raise ValueError("read_ply: only triangle faces are read")
            offset += dt.itemsize * count
            out["faces"] = f["v"].astype(np.int32)
        else:
            raise ValueError("read_ply: element %r is not read (only vertex and face)" % name)
    if "points" not in out:
        raise ValueError("read_ply: no vertex element")
    return out


MAX_CLOUD_POINTS = 2 ** 31 - 1
MAX_CELLS_PER_AXIS = 2 ** 21
NN_CELLS_PER_POINT = 2                      # the nearest-neighbour table's cells per indexed point, at most
NN_MAX_CELLS = 2 ** 26                      # and at most this many cells (two int32 tables of 256 MiB)


def _cloud(points, device, name):
    """A point set as contiguous device float32 [N,3] (one upload for host tensors and numpy arrays)"""
    if not torch.is_tensor(points):
        points = torch.from_numpy(np.ascontiguousarray(np.asarray(points)))
    if points.dim() != 2 or points.shape[1] != 3:
        raise ValueError("%s: expected points [N,3], got %s" % (name, list(points.shape)))
    if points.dtype != torch.float32:
        raise ValueError("%s: expected float32 points, got %s" % (name, points.dtype))
    if points.shape[0] > MAX_CLOUD_POINTS:
        raise ValueError("%s: at most 2^31 - 1 points" % name)
    return points.to(device).contiguous()


def _boxes(clouds, name):
    """The per-axis [min, max] of each non-empty set, read by the host in one read (None for an empty set); a
    non-finite coordinate anywhere makes a bound non-finite and is refused"""
    live = [c for c in clouds if c.shape[0]]
    vals = torch.cat([torch.cat((c.amin(0), c.amax(0))) for c in live]).tolist() if live else []
    if not all(math.isfinite(v) for v in vals):
        raise ValueError("%s: point coordinates must be finite" % name)
    boxes, k = [], 0
    for c in clouds:
        boxes.append((vals[k:k + 3], vals[k + 3:k + 6]) if c.shape[0] else None)
        k += 6 if c.shape[0] else 0
    return boxes


def nn_grid(lo, hi, n):
    """The nearest-neighbour table of n points in the box [lo, hi]: origin lo, the least cell size c (to a bisection's
    precision) with prod(max(1, ceil(extent / c))) cells at most min(NN_CELLS_PER_POINT n, NN_MAX_CELLS) and at most 2^21
    per axis, and dims.  A larger box (far floaters) gives larger cells, not a larger table; the search is exact for any."""
    lo = [float(v) for v in lo]
    ext = [max(0.0, float(b) - float(a)) for a, b in zip(lo, hi)]
    m = max(ext)
    if m == 0.0:
        return lo, 1.0, (1, 1, 1)
    cap = min(max(NN_CELLS_PER_POINT * n, 1), NN_MAX_CELLS)

    def dims(c):
        return tuple(max(1, math.ceil(e / c)) for e in ext)

    a, b = m / MAX_CELLS_PER_AXIS * (1 + 1e-9), m
    if math.prod(dims(a)) > cap:
        for _ in range(64):
            mid = math.sqrt(a * b)
            a, b = (a, mid) if math.prod(dims(mid)) <= cap else (mid, b)
        a = b
    return lo, a, dims(a)


class _Table:
    """The cell table of an indexed point set on the device (um_cloud_keys, a stable sort, um_cloud_ranges)"""

    def __init__(self, points, box):
        self.origin, self.cell, self.dims = nn_grid(box[0], box[1], points.shape[0])
        keys = _OPS.cloud_keys(points, self.origin, self.cell, self.dims)
        skeys, order = torch.sort(keys, stable=True)
        self.start, self.end, self.sorted = _OPS.cloud_ranges(skeys, order, points, self.dims)

    def nearest(self, queries):
        return _OPS.cloud_nearest(queries, self.sorted, self.start, self.end, self.origin, self.cell)

    def partials(self, queries, threshold):
        return _OPS.cloud_nearest_partials(queries, self.sorted, self.start, self.end, self.origin, self.cell, threshold)


def down_sample_grid(box, voxel_size, name):
    """Open3D's voxel grid of a set with bounds box = (min, max): origin min - v / 2 (float64), dims floor((max - origin)
    / v) + 1; more than 2^21 cells on an axis is refused"""
    v = float(voxel_size)
    origin = [float(a) - v / 2 for a in box[0]]
    dims = [math.floor((float(b) - o) / v) + 1 for b, o in zip(box[1], origin)]
    if max(dims) > MAX_CELLS_PER_AXIS:
        raise ValueError("%s: a %s-cell box at voxel size %g is more than 2^21 cells on an axis" % (name, dims, v))
    return origin, v, dims


def _down_sample_begin(points, box, voxel_size, name):
    origin, v, dims = down_sample_grid(box, voxel_size, name)
    skeys, order = torch.sort(_OPS.cloud_keys(points, origin, v, dims), stable=True)
    return skeys, order, _OPS.cloud_down_sample_count(skeys)


def _check_voxel(voxel_size, name):
    if isinstance(voxel_size, bool) or not isinstance(voxel_size, (int, float)) \
            or not (math.isfinite(voxel_size) and voxel_size > 0):
        raise ValueError("%s: voxel size must be positive and finite" % name)


@torch.no_grad()
def voxel_down_sample(points, voxel_size, device="cuda"):
    """Open3D's `VoxelDownSample` on the device: the points [N,3] (float32; a device tensor, a host tensor or a numpy
    array, uploaded once) binned into cells of `voxel_size` whose grid starts half a cell below the set's minimum, each
    occupied cell giving the mean of its points (float64 sums in input order, rounded to float32).  Returns float32 [M,3]
    on the device, ordered by cell (x fastest).  Host reads: the bounding box and the cell count M.  Non-finite
    coordinates and boxes of more than 2^21 cells per axis are refused with ValueError."""
    name = "voxel_down_sample"
    _check_voxel(voxel_size, name)
    dev = points.device if torch.is_tensor(points) and points.is_cuda else torch.device(device)
    p = _cloud(points, dev, name)
    with torch.cuda.device(dev):
        if p.shape[0] == 0:
            return p.new_zeros((0, 3))
        box, = _boxes([p], name)
        skeys, order, offsets = _down_sample_begin(p, box, voxel_size, name)
        return _OPS.cloud_down_sample(skeys, order, p, offsets, int(offsets[-1].item()))


@torch.no_grad()
def nearest_neighbors(queries, points, device="cuda"):
    """The exact nearest neighbour of every query among `points`, on the device: (distance float32 [Q], index int64 [Q]).
    The squared distance is float32 in one order, dx = q.x - p.x, ...; s = fmaf(dz, dz, fmaf(dy, dy, dx * dx)); the
    neighbour is the point of least s, ties to the least index, and the distance is sqrtf(s) correctly rounded: a
    brute-force float32 scan's result bit for bit, found by a ring search over a uniform grid whose pruning is proved
    conservative under that rounding (include/unimatch_sm100.h).  Both sets are float32 [N,3] device tensors, host
    tensors or numpy arrays (host sets are uploaded once).  Host reads: the bounding boxes (one read).  Empty `points`
    and non-finite coordinates are refused with ValueError; no queries give empty outputs."""
    name = "nearest_neighbors"
    dev = points.device if torch.is_tensor(points) and points.is_cuda else torch.device(device)
    q, p = _cloud(queries, dev, name), _cloud(points, dev, name)
    with torch.cuda.device(dev):
        if p.shape[0] == 0:
            raise ValueError("%s: no points to search" % name)
        _, box = _boxes([q, p], name)
        if q.shape[0] == 0:
            return q.new_zeros((0,)), torch.zeros((0,), dtype=torch.int64, device=dev)
        return _Table(p, box).nearest(q)


MAX_MESH_VIEWS = 65535
MAX_BIN_ENTRIES = 2 ** 31 - 1


def _camera(K, name):
    fx, fy, cx, cy = (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))
    if not (all(math.isfinite(v) for v in (fx, fy, cx, cy)) and fx != 0 and fy != 0):
        raise ValueError("%s: fx, fy, cx and cy must be finite, fx and fy nonzero" % name)
    return fx, fy, cx, cy


def _views(poses, name):
    ps = [_pose44(p, name) for p in poses]
    if not all(np.isfinite(p).all() for p in ps):
        raise ValueError("%s: camera poses must be finite" % name)
    if len(ps) > MAX_MESH_VIEWS:
        raise ValueError("%s: at most 65535 cameras per call" % name)
    return ps


def _faces(faces, dev, name):
    """Faces [T,3] of any integer type as a device tensor of that type (one upload for host data)"""
    if not torch.is_tensor(faces):
        faces = torch.from_numpy(np.ascontiguousarray(np.asarray(faces)))
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype.is_floating_point or faces.dtype.is_complex \
            or faces.dtype == torch.bool:
        raise ValueError("%s: expected integer faces [T,3], got %s %s" % (name, faces.dtype, list(faces.shape)))
    if faces.shape[0] > MAX_MESH_INDEX:
        raise ValueError("%s: at most 2^31 - 1 faces" % name)
    return faces.to(dev)


@torch.no_grad()
def render_mesh(points, faces, intrinsics, poses, frame_size, colors=None, near=0.01, far=None, device="cuda"):
    """Rasterise a triangle mesh on the device from N pinhole cameras: points float32 [P,3] and integer faces [T,3]
    (device tensors, host tensors or numpy arrays, host data uploaded once; the form `TSDFVolume.extract_mesh` returns
    and `read_ply` reads), intrinsics [3,3] at `frame_size` = (H, W), host camera-to-world poses [N,4,4] (as `render()`
    and `fuse_depths` take them), optional uint8 vertex `colors` [P,3].  Pixel (x, y) casts the ray through its centre,
    ((x - cx) / fx, (y - cy) / fy, 1) in camera coordinates; every face is two-sided, and the pixel takes the face hit at
    the least camera z-depth t with near <= t <= far (None: no limit), ties to the least face index.  Edge functions are
    evaluated from each edge's canonical vertex order, so faces sharing an edge leave no gap between them and a closed
    mesh around the camera has no miss.  Every operation, the pixel rectangle a face is restricted to and the tie rule
    are stated in include/unimatch_sm100.h (um_mesh_*); the result is the same from run to run.  Returns on the device
    {'depth': float32 [N,H,W] camera z-depth, 0 for a miss (`render()`'s convention, which `fuse_depths`, `track` and
    `depth_to_image` take), 'face': int32 [N,H,W] face index, -1 for a miss, and with `colors`, 'color': uint8 [N,H,W,3]
    (the vertex colours at the hit's perspective-correct barycentrics)}.  An empty mesh gives all misses and no cameras
    empty tensors.  Host reads: the vertices' bounds and the face-index range (one read), then the number of tile
    entries (one read), so `render_mesh` cannot be captured in a CUDA graph.  Non-finite vertices, face indices outside
    [0, P), bad intrinsics or poses, near <= 0 or far <= near, more than 65535 cameras, more than 2^31 - 1 pixels per
    frame and more than 2^31 - 1 tile entries are refused with ValueError, before the outputs are allocated."""
    name = "render_mesh"
    dev = points.device if torch.is_tensor(points) and points.is_cuda else torch.device(device)
    K = _intrinsics33(intrinsics, name)
    fx, fy, cx, cy = _camera(K, name)
    ps = _views(poses, name)
    h, w = (int(v) for v in frame_size)
    if h < 1 or w < 1 or h * w > MAX_VOXELS:
        raise ValueError("%s: frame_size must be (H, W) with at most 2^31 - 1 pixels" % name)
    with np.errstate(over="ignore"):
        near = _f32(near) if math.isfinite(near) else math.nan
        far = math.inf if far is None else (_f32(far) if not math.isnan(far) else math.nan)
    if not (math.isfinite(near) and near > 0 and far > near):
        raise ValueError("%s: near must be finite and > 0 in float32, far None or greater than near" % name)
    p = _cloud(points, dev, name)
    f = _faces(faces, dev, name)
    col = None
    if colors is not None:
        col = colors if torch.is_tensor(colors) else torch.from_numpy(np.ascontiguousarray(np.asarray(colors)))
        if col.dtype != torch.uint8 or tuple(col.shape) != (p.shape[0], 3):
            raise ValueError("%s: colors must be uint8 [P,3], one per point" % name)
        col = col.to(dev).contiguous()
    n_points, n_faces, n = p.shape[0], f.shape[0], len(ps)
    bounds = []
    if n_points:
        bounds += [p.amin(0).double(), p.amax(0).double()]
    if n_faces:
        bounds += [f.amin().double().reshape(1), f.amax().double().reshape(1)]
    vals = torch.cat(bounds).tolist() if bounds else []                  # the one host read of the inputs
    if n_points and not all(math.isfinite(v) for v in vals[:6]):
        raise ValueError("%s: vertex coordinates must be finite" % name)
    if n_faces and not (vals[-2] >= 0 and vals[-1] < n_points):
        raise ValueError("%s: face indices must lie in [0, %d)" % (name, n_points))
    if dev.type != "cuda":
        raise ValueError("%s: the mesh is rendered on a CUDA device" % name)
    with torch.cuda.device(dev):
        if n == 0 or n_faces == 0:                                    # no camera, or every pixel a miss
            out = {"depth": torch.zeros((n, h, w), dtype=torch.float32, device=dev),
                   "face": torch.full((n, h, w), -1, dtype=torch.int32, device=dev)}
            if col is not None:
                out["color"] = torch.zeros((n, h, w, 3), dtype=torch.uint8, device=dev)
            return out
        fi = f.to(torch.int32).contiguous()
        w2c = torch.from_numpy(_world_to_camera(ps)).to(dev)
        cam = (h, w, fx, fy, cx, cy, near, far)
        offsets = _OPS.mesh_bin_count(p, fi, w2c, *cam)
        n_entries = int(offsets[-1].item())
        if n_entries > MAX_BIN_ENTRIES:
            raise ValueError("%s: %d tile entries is more than 2^31 - 1 (fewer cameras or faces per call)"
                             % (name, n_entries))
        if n_entries:
            keys, values = _OPS.mesh_bin(p, fi, w2c, *cam, offsets, n_entries)
            del offsets
            keys, order = torch.sort(keys, stable=True)
        else:
            keys = order = values = torch.zeros((0,), dtype=torch.int64, device=dev)
        start, end = _OPS.mesh_ranges(keys, n, h, w)
        del keys
        depth, face, rgb = _OPS.mesh_raster(p, fi, col, w2c, *cam, order, values, start, end)
    out = {"depth": depth, "face": face}
    if col is not None:
        out["color"] = rgb
    return out


@torch.no_grad()
def visible_points(points, depths, intrinsics, poses, tolerance=0.05):
    """Which points some camera saw: bool [P] on the depths' device.  points float32 [P,3] (a device tensor, a host
    tensor or a numpy array, uploaded once), depths device float32 [N,H,W] (e.g. `render_mesh` of a reference mesh,
    sensor depths or `TSDFVolume.render`), intrinsics [3,3] at (H, W) and host camera-to-world poses [N,4,4].  Each view
    in order transforms and projects the point exactly as `fuse_depths` projects a voxel (camera z > 0, the nearest pixel
    inside the frame) and sees it iff that pixel's depth D is finite, D > 0 and z <= D + tolerance (float32).  A point
    with a non-finite coordinate is seen by no view.  One thread per point, no atomics (um_visible_points).  Culling for
    the 3D metrics is then plain indexing: `reconstruction_metrics(pred[vis_pred], gt[vis_gt])`.  The default tolerance
    is the metrics' default threshold: an occluder closer in depth than that hardly moves them."""
    name = "visible_points"
    if not (torch.is_tensor(depths) and depths.is_cuda and depths.dtype == torch.float32 and depths.dim() == 3):
        raise ValueError("%s: depths must be a device float32 tensor [N,H,W]" % name)
    n, h, w = depths.shape
    if h * w > MAX_VOXELS:
        raise ValueError("%s: at most 2^31 - 1 pixels per depth map" % name)
    K = _intrinsics33(intrinsics, name)
    fx, fy, cx, cy = _camera(K, name)
    ps = _views(poses, name)
    if len(ps) != n:
        raise ValueError("%s: %d depth maps need %d poses, got %d" % (name, n, n, len(ps)))
    if isinstance(tolerance, bool) or not isinstance(tolerance, (int, float)) or not math.isfinite(tolerance) \
            or tolerance < 0:
        raise ValueError("%s: tolerance must be finite and >= 0" % name)
    dev = depths.device
    p = _cloud(points, dev, name)
    with torch.cuda.device(dev):
        if n == 0 or p.shape[0] == 0:
            return torch.zeros((p.shape[0],), dtype=torch.bool, device=dev)
        w2c = torch.from_numpy(_world_to_camera(ps)).to(dev)
        return _OPS.visible_points(p, depths.contiguous(), w2c, fx, fy, cx, cy, _f32(tolerance))


MAX_CONSISTENCY_SOURCES = 255               # views is uint8


def sequence_sources(n, before, after):
    """The sources table of a clip of n frames for `filter_depths`: host int32 [n, before + after], row t listing frames
    t - 1, ..., t - before, then t + 1, ..., t + after, with -1 (no source) beyond the ends of the clip."""
    for v, nm in ((n, "n"), (before, "before"), (after, "after")):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 0:
            raise ValueError("sequence_sources: %s must be a non-negative int" % nm)
    t = np.arange(n)[:, None]
    offsets = np.array([-k for k in range(1, before + 1)] + list(range(1, after + 1)), np.int64)
    src = t + offsets[None, :]
    return np.where((src >= 0) & (src < n), src, -1).astype(np.int32).reshape(n, before + after)


def _positive_f32(v, name, what):
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
        raise ValueError("%s: %s must be positive and finite" % (name, what))
    with np.errstate(over="ignore"):
        f = _f32(v)
    if not (math.isfinite(f) and f > 0):
        raise ValueError("%s: %s must be positive and finite in float32" % (name, what))
    return f


def _consistency_args(n, sources, max_pixel, max_relative, min_views, name):
    """(sources int32 [n, S], max_pixel, max_relative, min_views) checked: S 1 .. 255, entries in [-1, n) and never the
    row's own frame, thresholds positive and finite in float32, min_views an int in [1, S]"""
    src = np.asarray(sources)
    if src.ndim != 2 or src.shape[0] != n or src.dtype.kind not in "iu":
        raise ValueError("%s: sources must be an integer table [N, S] with one row per depth map" % name)
    s = src.shape[1]
    if not 1 <= s <= MAX_CONSISTENCY_SOURCES:
        raise ValueError("%s: %d sources per frame; 1 .. 255 (the counts are uint8)" % (name, s))
    if src.size and (src.min() < -1 or src.max() >= n):
        raise ValueError("%s: source indices must lie in [-1, %d)" % (name, n))
    if (src == np.arange(n)[:, None]).any():
        raise ValueError("%s: a frame cannot be its own source" % name)
    if isinstance(min_views, bool) or not isinstance(min_views, (int, np.integer)) or not 1 <= min_views <= s:
        raise ValueError("%s: min_views must be an int in [1, %d]" % (name, s))
    return (src.astype(np.int32), _positive_f32(max_pixel, name, "max_pixel"),
            _positive_f32(max_relative, name, "max_relative"), int(min_views))


def _depth_stack(depths, name):
    if not (torch.is_tensor(depths) and depths.is_cuda and depths.dtype == torch.float32 and depths.dim() == 3):
        raise ValueError("%s: depths must be a device float32 tensor [N,H,W]" % name)
    n, h, w = depths.shape
    if h * w > MAX_VOXELS:
        raise ValueError("%s: at most 2^31 - 1 pixels per depth map" % name)
    if n > MAX_MESH_VIEWS:
        raise ValueError("%s: at most 65535 depth maps per call" % name)
    return n


@torch.no_grad()
def filter_depths(depths, intrinsics, poses, sources, max_pixel=1.0, max_relative=0.01, min_views=2):
    """Multi-view geometric consistency of N depth maps (MVSNet's check), on the device: device depths [N,H,W] (metric
    z-depth; zero, negative and non-finite depths are invalid), intrinsics [3,3] at (H, W), host camera-to-world poses
    [N,4,4] (as `fuse_depths` takes them) and a host sources table [N,S] (e.g. `sequence_sources`; -1 is no source).
    Every frame is a reference: each valid pixel is reprojected into each of its sources at its depth, the source depth
    is sampled there bilinearly (all four taps valid, inside the frame), and that point is reprojected back; the source
    is consistent when the pixel lands within `max_pixel` pixels of where it started and within `max_relative` of its
    depth.  The arithmetic is stated in include/unimatch_sm100.h (um_depth_consistency).  Returns on the device
    {'depth': fp32 [N,H,W], the depth where at least `min_views` sources are consistent and 0 (no estimate, which
    `fuse_depths` skips) elsewhere, 'views': uint8 [N,H,W] the number of consistent sources}.  One upload and one
    launch; no atomics, the same result from run to run.  A source equal to its own frame, indices outside [-1, N),
    more than 255 sources, bad cameras, poses and thresholds are refused with ValueError."""
    name = "filter_depths"
    n = _depth_stack(depths, name)
    _, h, w = depths.shape
    K = _intrinsics33(intrinsics, name)
    fx, fy, cx, cy = _camera(K, name)
    ps = _views(poses, name)
    if len(ps) != n:
        raise ValueError("%s: %d depth maps need %d poses, got %d" % (name, n, n, len(ps)))
    src, max_pixel, max_relative, min_views = _consistency_args(n, sources, max_pixel, max_relative, min_views, name)
    dev = depths.device
    if n == 0:
        return {"depth": depths.new_zeros((0, h, w)), "views": torch.zeros((0, h, w), dtype=torch.uint8, device=dev)}
    packed = np.concatenate([_camera_to_world(ps).view(np.uint8).ravel(), _world_to_camera(ps).view(np.uint8).ravel(),
                             np.arange(n, dtype=np.int32).view(np.uint8), src.view(np.uint8).ravel()])
    with torch.cuda.device(dev):
        buf = torch.from_numpy(packed).to(dev)                              # the one upload
        rows = buf[:96 * n].view(torch.float32).view(2, n, 3, 4)
        refs = buf[96 * n:100 * n].view(torch.int32)
        table = buf[100 * n:].view(torch.int32).view(n, src.shape[1])
        views, depth = _OPS.depth_consistency(depths.contiguous(), rows[0], rows[1], refs, table, fx, fy, cx, cy,
                                              max_pixel, max_relative, min_views)
    return {"depth": depth, "views": views}


@torch.no_grad()
def depth_points(depths, frames, intrinsics, poses):
    """The valid depths of N frames as a coloured world point cloud, on the device: device depths [N,H,W] (zero, negative
    and non-finite depths are skipped, so `filter_depths`' output gives the kept pixels), device uint8 frames [N,H,W,3],
    intrinsics [3,3] at (H, W) and host camera-to-world poses [N,4,4].  Each pixel is back-projected along the ray through
    its centre, exactly as `filter_depths` does.  Returns (points fp32 [P,3], colors uint8 [P,3]), ordered by frame, then
    row-major pixel: the form `write_ply` and `reconstruction_metrics` take.  A count pass, an ordered scan and a write
    pass, with one host read of P; more than 2^31 - 1 points is refused with ValueError before the outputs are
    allocated."""
    name = "depth_points"
    n = _depth_stack(depths, name)
    _, h, w = depths.shape
    if not (torch.is_tensor(frames) and frames.is_cuda and frames.dtype == torch.uint8
            and tuple(frames.shape) == tuple(depths.shape) + (3,) and frames.device == depths.device):
        raise ValueError("%s: frames must be device uint8 [N,H,W,3] at the depths' size, on their device" % name)
    K = _intrinsics33(intrinsics, name)
    fx, fy, cx, cy = _camera(K, name)
    ps = _views(poses, name)
    if len(ps) != n:
        raise ValueError("%s: %d depth maps need %d poses, got %d" % (name, n, n, len(ps)))
    dev = depths.device
    with torch.cuda.device(dev):
        if n == 0:
            return depths.new_zeros((0, 3)), torch.zeros((0, 3), dtype=torch.uint8, device=dev)
        d = depths.contiguous()
        c2w = torch.from_numpy(_camera_to_world(ps)).to(dev)
        offsets = _OPS.depth_points_count(d)
        total = int(offsets[-1].item())
        if total > MAX_CLOUD_POINTS:
            raise ValueError("%s: %d valid depths is more than 2^31 - 1 points (fewer frames per call)" % (name, total))
        return _OPS.depth_points(d, frames.contiguous(), c2w, fx, fy, cx, cy, offsets, total)
