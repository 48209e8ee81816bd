"""Leaderboard submissions: the reference's `--submission` drivers (evaluate_flow.py:19-156, evaluate_stereo.py:28-298) on
batches, with each file's payload encoded on the device and the files written by a pool of host threads.

`create_flow_submission` writes Sintel `.flo` files and KITTI 16-bit flow PNGs, `create_stereo_submission` KITTI 16-bit
disparity PNGs and ETH3D / Middlebury `.pfm` files with their runtime files, in the reference's directory layout.  Samples
of equal size are grouped into batches of `batch` (one open batch per size, flushed when full and at the end, as the
validation drivers do), padded with the reference's `InputPadder` mode or resized to `inference_size`, and run through the
model.  One `um_encode_submission` launch per batch turns the model's output into every sample's file payload: the unpad
crop or the resize back with the reference's two-step rescale, then the format's bytes -- float32 for `.flo` / `.pfm`,
PNG scanlines with the "Up" filter already applied for the PNGs.  Only that buffer is downloaded, into one of two pinned
buffers; a `ThreadPoolExecutor` of `writers` threads waits for the copy, deflates PNG scanlines (zlib level 1, Z_RLE; zlib
releases the GIL), adds the header and writes the file.  A batch waits for the writers of the batch that last used its
pinned buffer, so host memory stays bounded; an error in a writer is raised in the caller; every file is complete and closed
when the function returns.

The PNG container comes from the small stdlib writer below (no cv2, skimage or imageio); `oracle/submission_io.py` states
every payload and header in numpy.
"""
import os
import struct
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import ops
from .evaluation import _upload
from .inference import InputPadder, _resize, disparity_to_image, flow_to_image

_OPS = torch.ops.unimatch_sm100

PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
FLO_TAG = b"PIEH"               # writeFlow's TAG_CHAR, np.array([202021.25], np.float32)
WARMUP_FORWARDS = 5             # evaluate_stereo.py:147-157, :243-253


# ---- file formats ------------------------------------------------------------------------------------------------------
def deflate(scanlines):
    """zlib stream of filtered PNG scanlines: level 1 with the Z_RLE strategy."""
    c = zlib.compressobj(1, zlib.DEFLATED, 15, 8, zlib.Z_RLE)
    return c.compress(scanlines) + c.flush()


def _chunk(kind, body):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))


def png_bytes(scanlines, h, w, bit_depth, colour_type):
    """A PNG file around filtered scanlines (each row a filter byte, then its samples big-endian): signature, IHDR, one
    IDAT, IEND.  colour_type 0 = grey, 2 = RGB."""
    ihdr = struct.pack(">IIBBBBB", w, h, bit_depth, colour_type, 0, 0, 0)
    return PNG_SIGNATURE + _chunk(b"IHDR", ihdr) + _chunk(b"IDAT", deflate(scanlines)) + _chunk(b"IEND", b"")


def picture_scanlines(rgb):
    """uint8 [H, W, 3] RGB -> unfiltered scanlines (filter byte 0 on every row)."""
    h = rgb.shape[0]
    rows = np.empty((h, 1 + rgb.shape[1] * 3), dtype=np.uint8)
    rows[:, 0] = 0
    rows[:, 1:] = rgb.reshape(h, -1)
    return rows.tobytes()


def flo_header(h, w):
    return FLO_TAG + struct.pack("<ii", w, h)


def pfm_header(h, w):
    """write_pfm's header for a little-endian greyscale image (utils/file_io.py:110-123)."""
    return b"Pf\n" + b"%d %d\n" % (w, h) + b"%f\n" % -1


# ---- batching and the writer pool ------------------------------------------------------------------------------------------
def _batches(samples, batch, shape_of):
    """Lists of samples of equal `shape_of(sample)`, at most `batch` long: one open batch per shape, flushed when full and,
    at the end, in the order the shapes were first opened."""
    if batch < 1:
        raise ValueError("batch must be positive")
    open_batches = {}
    for s in samples:
        key = shape_of(s)
        open_batches.setdefault(key, []).append(s)
        if len(open_batches[key]) == batch:
            yield open_batches.pop(key)
    for key in list(open_batches):
        yield open_batches.pop(key)


class _WriterPool:
    """Two pinned staging slots and a pool of writer threads.  `stage` waits for the writers of the batch that last used the
    slot (re-raising their errors), copies device tensors into the slot and records an event; jobs wait on that event."""

    def __init__(self, writers, cuda):
        if writers < 1:
            raise ValueError("writers must be positive")
        self.cuda = cuda
        self.pool = ThreadPoolExecutor(max_workers=writers, thread_name_prefix="submission-writer")
        self.slots = [{"buffers": {}, "futures": []} for _ in range(2)]
        self.next = 0
        self.busy_s = 0.0                  # summed wall time of the jobs (writer occupancy = busy_s / (writers * elapsed))
        self.d2h_bytes = 0

    def _drain(self, slot):
        futures, slot["futures"] = slot["futures"], []
        for f in futures:
            self.busy_s += f.result()

    def stage(self, tensors):
        slot = self.slots[self.next]
        self.next ^= 1
        self._drain(slot)
        host = {}
        for name, t in tensors.items():
            self.d2h_bytes += t.numel() * t.element_size()
            if not t.is_cuda:
                host[name] = t.numpy()
                continue
            buf = slot["buffers"].get(name)
            if buf is None or buf.dtype != t.dtype or buf.numel() < t.numel():
                buf = torch.empty((t.numel(),), dtype=t.dtype, pin_memory=True)
                slot["buffers"][name] = buf
            h = buf[:t.numel()].view(t.shape)
            h.copy_(t, non_blocking=True)
            host[name] = h.numpy()
        ready = None
        if self.cuda:
            ready = torch.cuda.Event()
            ready.record()
        return slot, host, ready

    def submit(self, slot, ready, fn, *args):
        def job():
            t0 = time.perf_counter()
            if ready is not None:
                ready.synchronize()
            fn(*args)
            return time.perf_counter() - t0
        slot["futures"].append(self.pool.submit(job))

    def close(self, error=None):
        """Wait for every job; re-raise the first writer error unless the caller is already raising one."""
        try:
            if error is None:
                for slot in self.slots:
                    self._drain(slot)
        finally:
            self.pool.shutdown(wait=True, cancel_futures=error is not None)


def _write(path, *parts):
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "wb") as f:
        for p in parts:
            f.write(p)


def _write_png(path, scanlines, h, w, bit_depth, colour_type):
    _write(path, png_bytes(scanlines, h, w, bit_depth, colour_type))


def _write_picture(path, rgb):
    _write_png(path, picture_scanlines(rgb), rgb.shape[0], rgb.shape[1], 8, 2)


class _ModelTimer:
    """Time of one model call: CUDA events on a CUDA device (read by the writer thread once the call has run), the host
    clock otherwise."""

    def __init__(self, cuda):
        self.cuda = cuda
        if cuda:
            self.start, self.end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def __enter__(self):
        if self.cuda:
            self.start.record()
        else:
            self.t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        if self.cuda:
            self.end.record()
        else:
            self.elapsed = time.perf_counter() - self.t0

    def seconds(self):
        if not self.cuda:
            return self.elapsed
        self.end.synchronize()
        return self.start.elapsed_time(self.end) / 1000.0


def _write_runtime(path, prefix, timer, n):
    """The sample's share of its batch's model time, in seconds, as str(float) after `prefix`."""
    _write(path, (prefix + str(timer.seconds() / n)).encode())


# ---- geometry ------------------------------------------------------------------------------------------------------------
def _geometry(task, protocol, ori, padding_factor, inference_size):
    """How the reference driver brings a sample to the model and back: ('pad', mode) -- InputPadder and its unpad --,
    ('resize', size) -- resize to `size` and back with the rescale, even at the original size, as the reference does --
    or ('none', None) for ETH3D at a size that is already a multiple (evaluate_stereo.py:133-145, :178-181)."""
    if task == "stereo" and protocol == "eth3d":
        if inference_size is None:
            size = (-(-ori[0] // padding_factor) * padding_factor, -(-ori[1] // padding_factor) * padding_factor)
        else:
            size = (int(inference_size[0]), int(inference_size[1]))
        return ("none", None) if size == ori else ("resize", size)
    if inference_size is not None:
        if len(inference_size) != 2:
            raise ValueError("inference_size must be (height, width)")
        return "resize", (int(inference_size[0]), int(inference_size[1]))
    return "pad", "kitti" if (task, protocol) == ("flow", "kitti") else "sintel"


def _prepare(images, geom, padding_factor):
    """The model's inputs and the encode geometry (resize, top, left) for stacked device images [B, 3, H, W]."""
    kind, arg = geom
    if kind == "pad":
        padder = InputPadder(images[0].shape, mode=arg, padding_factor=padding_factor)
        left, _, top, _ = padder._pad
        return [x.contiguous() for x in padder.pad(*images)], (False, top, left)
    if kind == "resize":
        return [_resize(x, arg) for x in images], (True, 0, 0)
    return [x.float().contiguous() for x in images], (False, 0, 0)


def _encode(pred, fmt, ori, enc):
    resize, top, left = enc
    return _OPS.encode_submission(pred.float().contiguous(), fmt, int(ori[0]), int(ori[1]), bool(resize), int(top), int(left))


def _run_batches(batches, writers, device, run):
    """Runs every batch through `run(pool, items)`; returns {'samples', 'batches', 'd2h_bytes', 'writer_seconds'}."""
    pool = _WriterPool(writers, device.type == "cuda")
    samples = nb = 0
    try:
        for items in batches:
            run(pool, items)
            samples, nb = samples + len(items), nb + 1
    except BaseException as e:
        pool.close(error=e)
        raise
    pool.close()
    return {"samples": samples, "batches": nb, "d2h_bytes": pool.d2h_bytes, "writer_seconds": pool.busy_s}


# ---- drivers -------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def create_flow_submission(model, dataset, *, protocol, output_path, dstype="clean", batch=8, device="cuda", padding_factor=8,
                           inference_size=None, save_vis_flow=False, no_save_flo=False, writers=8, **model_kwargs):
    """evaluate_flow.py's `create_<protocol>_submission` on `dataset`, `protocol` 'sintel' or 'kitti'.

    * 'sintel': samples (img1, img2, (sequence, frame)) -> `output_path/dstype/sequence/frame%04d.flo` numbered frame + 1
      (unless `no_save_flo`), and the flow picture as the `.png` beside it with `save_vis_flow`.  InputPadder mode 'sintel'.
    * 'kitti': samples (img1, img2, (frame_id,)) -> the 16-bit flow PNG `output_path/frame_id`; with `save_vis_flow` the
      flow picture replaces it, as in the reference.  InputPadder mode 'kitti'.

    Images are float [3, H, W] in [0, 255].  With `inference_size` every pair is resized to it and the flow resized back,
    u scaled by (u * W) / w and v by (v * H) / h.  Pictures are `flow_to_image` of the written flow.  `model_kwargs` go to
    `model(...)` (attn_type, attn_splits_list, corr_radius_list, prop_radius_list, num_reg_refine)."""
    if protocol not in ("sintel", "kitti"):
        raise ValueError("create_flow_submission: protocol must be 'sintel' or 'kitti'")
    if model_kwargs.setdefault("task", "flow") != "flow":
        raise ValueError("create_flow_submission drives the flow task only")
    device = torch.device(device)
    sintel = protocol == "sintel"
    write_flow = not (no_save_flo if sintel else save_vis_flow)
    os.makedirs(output_path, exist_ok=True)

    def run(pool, items):
        ori = tuple(items[0][0].shape[-2:])
        geom = _geometry("flow", protocol, ori, padding_factor, inference_size)
        img1, img2 = (_upload(torch.stack([torch.as_tensor(s[k]) for s in items]), device) for k in (0, 1))
        (img1, img2), enc = _prepare([img1, img2], geom, padding_factor)
        pred = model(img1, img2, **model_kwargs)["flow_preds"][-1]
        out = {}
        if write_flow:
            out["payload"] = _encode(pred, ops.SUBMIT_FLO if sintel else ops.SUBMIT_KITTI_FLOW_PNG, ori, enc)
        if save_vis_flow:
            flo = out["payload"] if sintel and write_flow else _encode(pred, ops.SUBMIT_FLO, ori, enc)
            flow = flo.view(torch.float32).view(len(items), ori[0], ori[1], 2).permute(0, 3, 1, 2)
            out["picture"] = flow_to_image(flow.contiguous())
        slot, host, ready = pool.stage(out)
        h, w = ori
        for i, s in enumerate(items):
            if sintel:
                sequence, frame = s[2]
                path = os.path.join(output_path, dstype, sequence, "frame%04d.flo" % (int(frame) + 1))
                if write_flow:
                    pool.submit(slot, ready, _write, path, flo_header(h, w), host["payload"][i])
                if save_vis_flow:
                    pool.submit(slot, ready, _write_picture, path.replace(".flo", ".png"), host["picture"][i])
            else:
                path = os.path.join(output_path, s[2][0])
                if write_flow:
                    pool.submit(slot, ready, _write_png, path, host["payload"][i], h, w, 16, 2)
                else:
                    pool.submit(slot, ready, _write_picture, path, host["picture"][i])

    return _run_batches(_batches(dataset, batch, lambda s: tuple(np.shape(s[0]))), writers, device, run)


@torch.no_grad()
def create_stereo_submission(model, dataset, *, protocol, output_path, batch=8, device="cuda", padding_factor=16,
                             inference_size=None, save_vis_disp=False, writers=8, **model_kwargs):
    """evaluate_stereo.py's `create_<protocol>_submission` on `dataset`, `protocol` 'kitti', 'eth3d' or 'middlebury'.
    Samples are dicts with 'left', 'right' (ImageNet-normalised [3, H, W]) and 'left_name'.

    * 'kitti': the 16-bit disparity PNG `output_path/left_name`, uint16(256 d).  InputPadder mode 'sintel', or the resize
      to `inference_size` and back.  The reference writes no picture here, so `save_vis_disp` is refused.
    * 'eth3d': `<scene>.pfm` and `<scene>.txt` holding 'runtime <seconds>', scene = the directory name of 'left_name'.  The
      pair is resized to the nearest multiple of `padding_factor` (or to `inference_size`) only if that changes its size.
    * 'middlebury': `<scene>/disp0GMStereo.pfm` and `<scene>/timeGMStereo.txt` holding '<seconds>'.  InputPadder mode
      'sintel', or the resize.  Kept quirk (evaluate_stereo.py:262-268): the saved disparity comes from a forward without
      `num_reg_refine`, so the model's default (1) is used; the warm-up forwards do pass it.

    With `save_vis_disp` (ETH3D, Middlebury) `<scene>.png`, the `vis_disparity` picture, replaces the files, as in the
    reference.  Disparities resized back are scaled by (d * W) / w.

    Runtime: before the first batch the model runs the reference's 5 warm-up forwards on it; then each batch's model call is
    timed with CUDA events, and each sample's runtime is that time divided by the batch size.  With `batch=1` this is the
    reference's per-pair measurement (a host clock between two synchronisations there)."""
    if protocol not in ("kitti", "eth3d", "middlebury"):
        raise ValueError("create_stereo_submission: protocol must be 'kitti', 'eth3d' or 'middlebury'")
    if protocol == "kitti" and save_vis_disp:
        raise ValueError("create_stereo_submission: the KITTI submission has no picture (save_vis_disp)")
    if model_kwargs.setdefault("task", "stereo") != "stereo":
        raise ValueError("create_stereo_submission drives the stereo task only")
    device = torch.device(device)
    timed = protocol != "kitti"
    fwd_kwargs = {k: v for k, v in model_kwargs.items() if not (protocol == "middlebury" and k == "num_reg_refine")}
    warm = [timed]
    os.makedirs(output_path, exist_ok=True)

    def run(pool, items):
        ori = tuple(items[0]["left"].shape[-2:])
        geom = _geometry("stereo", protocol, ori, padding_factor, inference_size)
        left, right = (_upload(torch.stack([torch.as_tensor(s[k]) for s in items]), device) for k in ("left", "right"))
        (left, right), enc = _prepare([left, right], geom, padding_factor)
        if warm[0]:
            for _ in range(WARMUP_FORWARDS):
                model(left, right, **model_kwargs)
            warm[0] = False
        with _ModelTimer(device.type == "cuda") as timer:
            pred = model(left, right, **fwd_kwargs)["flow_preds"][-1].unsqueeze(1)
        n, (h, w) = len(items), ori
        out = {}
        if protocol == "kitti":
            out["payload"] = _encode(pred, ops.SUBMIT_KITTI_DISP_PNG, ori, enc)
        else:
            pfm = _encode(pred, ops.SUBMIT_PFM, ori, enc)
            if save_vis_disp:
                disp = pfm.view(torch.float32).view(n, h, w).flip(1)
                out["picture"] = disparity_to_image(disp.contiguous())
            else:
                out["payload"] = pfm
        slot, host, ready = pool.stage(out)
        for i, s in enumerate(items):
            scene = os.path.basename(os.path.dirname(s["left_name"]))
            if protocol == "kitti":
                pool.submit(slot, ready, _write_png, os.path.join(output_path, s["left_name"]), host["payload"][i], h, w, 16, 0)
            elif save_vis_disp:
                pool.submit(slot, ready, _write_picture, os.path.join(output_path, scene + ".png"), host["picture"][i][..., ::-1])
            elif protocol == "eth3d":
                pool.submit(slot, ready, _write, os.path.join(output_path, scene + ".pfm"), pfm_header(h, w), host["payload"][i])
                pool.submit(slot, ready, _write_runtime, os.path.join(output_path, scene + ".txt"), "runtime ", timer, n)
            else:
                d = os.path.join(output_path, scene)
                pool.submit(slot, ready, _write, os.path.join(d, "disp0GMStereo.pfm"), pfm_header(h, w), host["payload"][i])
                pool.submit(slot, ready, _write_runtime, os.path.join(d, "timeGMStereo.txt"), "", timer, n)

    return _run_batches(_batches(dataset, batch, lambda s: tuple(np.shape(s["left"]))), writers, device, run)
