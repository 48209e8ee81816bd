"""Drop-in inference commands: the reference's `inference_flow` (evaluate_flow.py:641-831), `inference_stereo`
(evaluate_stereo.py:711-843) and `inference_depth` (evaluate_depth.py:296-419), reading the same directories and videos and
writing the same files, with the pairs streamed through the runners.

    import main_flow, unimatch_b200
    main_flow.inference_flow = unimatch_b200.inference_flow     # then main_flow.main(args) as usual

Each driver takes the reference function's keyword arguments (so `main_*.py` calls it unchanged) and a few of its own with
defaults: `batch` (pairs per device step), `device`, `readers` (decode threads), `writers` (file-writer threads) and
`max_buckets` (inference sizes whose CUDA graphs are kept).  It returns a statistics dict (the reference
returns None): pairs, steps, bytes copied each way, and the summed busy seconds of the reader and writer threads.

* Reading: files are listed exactly as the reference lists them and decoded as it decodes them, on `readers` threads in
  input order, up to `readers + 2 * batch` items ahead of the runner (PIL and cv2 release the GIL while decoding).  A video
  is decoded by cv2 on one reader thread, frame after frame.
* Device work: `MixedSizeFlowRunner` (a directory: pairs of any size and orientation), `VideoFlowRunner` (a video: every
  frame encoded once), `MixedSizeStereoRunner`, and `DepthSequenceRunner` (a depth directory of one frame size: every
  frame encoded once) or `MixedSizeDepthRunner` (frames of several sizes), each with its pictures painted on the device.
* Writing: the runners hand out views of pinned staging that later steps reuse, so the main thread copies each result into
  its file layout (PNG scanlines, `.flo` interleaved u / v, `.pfm` rows bottom to top) and the `submission._WriterPool`
  threads deflate and write.  Every `batch` pairs the pool waits for the jobs of the group before last, so at most two
  groups of copies are held; a writer's error is raised in the caller, and every file is complete when the driver returns.
  `inference_flow(save_video=True)` encodes its mp4 with cv2's `mp4v` (MPEG-4 Part 2) on one ordered writer thread.  The
  reference writes H.264 through imageio / libx264, which this package does not depend on (and cv2's own builds often
  cannot encode H.264), so the video's pixels match the pictures up to the codec's loss, not the reference's bitstream.

Deliberate difference: the reference's `inference_flow` never resets its transpose flag (evaluate_flow.py:675, :714-717,
:757-758), so after the first portrait pair it transposes every later flow back, landscape ones included, and writes
wrongly shaped files.  Here each pair is transposed only when it is itself portrait.
"""
import collections
import itertools
import os
import time
from concurrent.futures import ThreadPoolExecutor
from glob import glob

import numpy as np
import torch
from PIL import Image

from .inference import (DepthSequenceRunner, MixedSizeDepthRunner, MixedSizeFlowRunner, MixedSizeStereoRunner,
                        VideoFlowRunner, _flow_outputs, _inference_size, _relative_poses, _resize, flow_to_image)
from .submission import _WriterPool, _write, _write_png, flo_header, pfm_header, picture_scanlines

# result key of the runner -> (file name suffix, encoding), in the order the reference writes them
FLOW_FILES = {"vis": ("_flow.png", "rgb"), "vis_bwd": ("_flow_bwd.png", "rgb"), "fwd_occ": ("_occ_fwd.png", "mask"),
              "bwd_occ": ("_occ_bwd.png", "mask"), "flow": ("_pred.flo", "flo"), "flow_bwd": ("_pred_bwd.flo", "flo")}
STEREO_FILES = {"disp": ("_disp.pfm", "pfm"), "vis": ("_disp.png", "bgr"), "disp_right": ("_disp_right.pfm", "pfm"),
                "vis_right": ("_disp_right.png", "bgr")}
DEPTH_FILES = {"vis": (".png", "rgb"), "vis_bwd": ("_bwd.png", "rgb")}


# ---- listing and naming (pure functions) -------------------------------------------------------------------------------
def _images(pattern_dir):
    return sorted(glob(pattern_dir + "/*.png") + glob(pattern_dir + "/*.jpg"))


def _stem(path):
    return os.path.basename(path)[:-4]


def flow_inputs(inference_dir):
    """The frames of a flow directory in the reference's order (evaluate_flow.py:680); pair t is (files[t], files[t + 1])."""
    return _images(inference_dir)


def flow_keys(pred_bidir_flow=False, fwd_bwd_consistency_check=False, save_flo_flow=False):
    """The result keys written for each pair (evaluate_flow.py:762-812)."""
    keys = ["vis"]
    if pred_bidir_flow:
        keys.append("vis_bwd")
        if fwd_bwd_consistency_check:
            keys += ["fwd_occ", "bwd_occ"]
    if save_flo_flow:
        keys += ["flow", "flow_bwd"] if pred_bidir_flow else ["flow"]
    return keys


def flow_prefix(files, t, video):
    """The name prefix of pair t: `%04d` for a video, else the first frame's name without its 4-character extension."""
    return "%04d" % t if video else _stem(files[t])


def stereo_inputs(inference_dir=None, inference_dir_left=None, inference_dir_right=None):
    """(left files, right files) as evaluate_stereo.py:739-751 lists them: the alternating files of one directory, or two
    sorted directories of equally many files."""
    if inference_dir is None and not (inference_dir_left and inference_dir_right):
        raise ValueError("inference_stereo needs inference_dir, or inference_dir_left and inference_dir_right")
    if inference_dir is not None:
        files = _images(inference_dir)
        left, right = files[::2], files[1::2]
    else:
        left, right = _images(inference_dir_left), _images(inference_dir_right)
    if len(left) != len(right):
        raise ValueError("inference_stereo: %d left images but %d right images" % (len(left), len(right)))
    return left, right


def stereo_keys(pred_bidir_disp=False, save_pfm_disp=False):
    """The result keys written for each pair (evaluate_stereo.py:815-841)."""
    keys = ["disp", "vis"] if save_pfm_disp else ["vis"]
    if pred_bidir_disp:
        keys += ["disp_right", "vis_right"] if save_pfm_disp else ["vis_right"]
    return keys


def depth_inputs(inference_dir):
    """(frames, pose files, intrinsics file) of a ScanNet-layout directory (evaluate_depth.py:327-334): color/*.jpg|png,
    pose/*.txt and the first file glob gives under intrinsic/."""
    imgs = sorted(glob(os.path.join(inference_dir, "color", "*.jpg")) + glob(os.path.join(inference_dir, "color", "*.png")))
    poses = sorted(glob(os.path.join(inference_dir, "pose", "*.txt")))
    intrinsics = glob(os.path.join(inference_dir, "intrinsic", "*.txt"))
    if not intrinsics:
        raise ValueError("inference_depth: no intrinsic/*.txt under %s" % inference_dir)
    if len(imgs) != len(poses):
        raise ValueError("inference_depth: %d frames but %d poses" % (len(imgs), len(poses)))
    return imgs, poses, intrinsics[0]


def depth_keys(pred_bidir_depth=False):
    return ["vis", "vis_bwd"] if pred_bidir_depth else ["vis"]


def output_names(files, keys, prefix):
    """{result key: file name} of one pair whose name prefix is `prefix`."""
    return {k: prefix + files[k][0] for k in keys}


# ---- reading -------------------------------------------------------------------------------------------------------------
def _header_size(path):
    """(height, width) from the image header, without decoding the pixels"""
    with Image.open(path) as img:
        w, h = img.size
    return h, w


def _flow_frame(path):
    """np.array(read_gen(f)).astype(np.uint8), grey tiled to 3 channels, alpha dropped (evaluate_flow.py:694-705)"""
    with Image.open(path) as img:
        a = np.array(img).astype(np.uint8)
    a = np.tile(a[..., None], (1, 1, 3)) if a.ndim == 2 else a[..., :3]
    return np.ascontiguousarray(a)


def _rgb_frame(path):
    """np.array(Image.open(f).convert('RGB')) (evaluate_stereo.py:766-767, evaluate_depth.py:342-343)"""
    with Image.open(path) as img:
        return np.array(img.convert("RGB"))


def _pose(path):
    return np.loadtxt(path, delimiter=" ").astype(np.float32).reshape((4, 4))


class _Readers:
    """fn(item) for every item, in input order, on `readers` threads, at most `ahead` items in flight; `busy_s` sums the
    threads' time inside fn."""

    def __init__(self, readers, ahead):
        if readers < 1:
            raise ValueError("readers must be positive")
        self.readers, self.ahead, self.busy_s = int(readers), max(int(ahead), int(readers)), 0.0

    def map(self, fn, items):
        def timed(x):
            t0 = time.perf_counter()
            out = fn(x)
            return out, time.perf_counter() - t0

        items = iter(items)
        with ThreadPoolExecutor(self.readers, thread_name_prefix="inference-reader") as pool:
            pending = collections.deque(pool.submit(timed, x) for x in itertools.islice(items, self.ahead))
            while pending:
                out, s = pending.popleft().result()
                self.busy_s += s
                pending.extend(pool.submit(timed, x) for x in itertools.islice(items, 1))
                yield out


def _consecutive(frames):
    """(frame t, frame t + 1) of a frame stream, each frame decoded once"""
    frames = iter(frames)
    prev = next(frames, None)
    for f in frames:
        yield prev, f
        prev = f


def _video_frames(path, readers):
    """The RGB frames of a video as utils/file_io.py:203-223 extracts them (cv2, BGR -> RGB), decoded one after the other
    on a reader thread a few frames ahead."""
    import cv2
    cap = cv2.VideoCapture(path)
    if not cap.isOpened():
        raise ValueError("inference_flow: cannot open the video %s" % path)

    def read(_):
        ok, img = cap.read()
        return cv2.cvtColor(img, cv2.COLOR_BGR2RGB) if ok else None

    frames = readers.map(read, itertools.count())
    try:
        for f in frames:
            if f is None:
                return
            yield f
    finally:
        frames.close()                       # waits for the reads in flight before the capture is released
        cap.release()


# ---- writing -------------------------------------------------------------------------------------------------------------
def _job(path, x, encoding):
    """A writer job for result `x` (a CPU view of reused staging): the copy into the file's layout happens here, on the
    caller's thread; the job deflates (PNG) and writes."""
    a = x.numpy()
    if encoding == "flo":                    # writeFlow: [H, W, 2] float32, u and v interleaved
        return _write, path, flo_header(a.shape[1], a.shape[2]), np.ascontiguousarray(a.transpose(1, 2, 0))
    if encoding == "pfm":                    # write_pfm: rows bottom to top
        return _write, path, pfm_header(*a.shape), np.ascontiguousarray(a[::-1])
    if encoding == "mask":                   # Image.fromarray((occ * 255.).astype(np.uint8)): 8-bit grey
        a, colour = (a * 255.).astype(np.uint8), 0
    elif encoding == "bgr":                  # cv2.imwrite of a BGR picture stores RGB
        a, colour = a[..., ::-1], 2
    else:
        colour = 2
    return (_write_png, path, picture_scanlines(a), a.shape[0], a.shape[1], 8, colour)


def video_frame(rgb):
    """A picture [H, W, 3] RGB as `cv2.VideoWriter` takes it: a BGR copy, with an odd height or width made even by
    repeating the last row or column (mp4v drops an odd last row or column)."""
    a = np.asarray(rgb)[..., ::-1]
    h, w = a.shape[:2]
    if h % 2 or w % 2:
        a = np.pad(a, ((0, h % 2), (0, w % 2), (0, 0)), mode="edge")
    return np.ascontiguousarray(a)


def video_name(inference_video, concat_flow_img):
    """The reference's video file name (evaluate_flow.py:815-816)."""
    return os.path.basename(inference_video)[:-4] + ("_flow_img.mp4" if concat_flow_img else "_flow.mp4")


class _VideoWriter:
    """The frames of one mp4 (cv2.VideoWriter, fourcc mp4v, at `fps`), written in order by one thread.  `submit` copies
    the picture (a view of reused staging) on the caller's thread; at most `ahead` frames wait for the writer."""

    def __init__(self, path, fps, ahead=16):
        self.path, self.fps, self.ahead = path, float(fps), int(ahead)
        self.pool = ThreadPoolExecutor(1, thread_name_prefix="video-writer")
        self.pending = collections.deque()
        self.writer, self.busy_s, self.frames = None, 0.0, 0

    def _write(self, frame):
        t0 = time.perf_counter()
        self.writer.write(frame)
        return time.perf_counter() - t0

    def submit(self, rgb):
        import cv2
        frame = video_frame(rgb)
        if self.writer is None:
            self.writer = cv2.VideoWriter(self.path, cv2.VideoWriter_fourcc(*"mp4v"), self.fps, (frame.shape[1], frame.shape[0]))
            if not self.writer.isOpened():
                raise RuntimeError("cannot open %s for writing with the mp4v codec" % self.path)
        self.pending.append(self.pool.submit(self._write, frame))
        self.frames += 1
        while len(self.pending) > self.ahead:
            self.busy_s += self.pending.popleft().result()

    def close(self, error=None):
        """Finish the file; re-raise a writer error unless the caller is already raising one."""
        try:
            if error is None:
                while self.pending:
                    self.busy_s += self.pending.popleft().result()
        finally:
            self.pool.shutdown(wait=True, cancel_futures=error is not None)
            if self.writer is not None:
                self.writer.release()


def _write_results(results, names, writers, group, video=None):
    """Writes every (index, result) of `results`, `names(index)` giving {key: (path, encoding)}, and with `video` each
    result's 'vis' as the next frame of that `_VideoWriter`; returns the writers' summed busy seconds."""
    pool = _WriterPool(writers, False)
    slot = pool.stage({})[0]
    n = 0
    try:
        for index, r in results:
            for key, (path, encoding) in names(index).items():
                pool.submit(slot, None, *_job(path, r[key], encoding))
            if video is not None:
                video.submit(r["vis"])
            n += 1
            if n % group == 0:
                slot = pool.stage({})[0]       # waits for the jobs of the group before last
    except BaseException as e:
        pool.close(error=e)
        if video is not None:
            video.close(error=e)
        raise
    pool.close()
    if video is not None:
        video.close()
        return pool.busy_s + video.busy_s
    return pool.busy_s


def _named(files, keys, output_path, prefix_of):
    def names(index):
        return {k: (os.path.join(output_path, name), files[k][1]) for k, name in output_names(files, keys, prefix_of(index)).items()}
    return names


def _sequence_stats(runner, pairs, extra_h2d=0):
    """What a sequence runner copied: the first frame, then per step its pinned inputs up and its pinned outputs down."""
    steps = -(-pairs // runner.batch)
    h2d = runner.h * runner.w * 3 + steps * (runner.pin[0].nbytes + extra_h2d)
    d2h = steps * sum(v.nbytes for v in runner.out_pin[0].values()) if pairs else 0
    return {"pairs": pairs, "steps": steps, "h2d_bytes": h2d if pairs else 0, "d2h_bytes": d2h}


def _stats(base, readers, writer_s):
    return dict(base, reader_seconds=readers.busy_s, writer_seconds=writer_s)


# ---- drivers -------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def inference_flow(model, inference_dir=None, inference_video=None, output_path="output", padding_factor=8,
                   inference_size=None, save_flo_flow=False, attn_type="swin", attn_splits_list=None, corr_radius_list=None,
                   prop_radius_list=None, num_reg_refine=1, pred_bidir_flow=False, pred_bwd_flow=False,
                   fwd_bwd_consistency_check=False, save_video=False, concat_flow_img=False, batch=8, device="cuda", readers=4,
                   writers=8, max_buckets=4):
    """`evaluate_flow.inference_flow` on a directory (consecutive pairs of its sorted *.png + *.jpg files, through
    `MixedSizeFlowRunner`, `max_frame_size` from the image headers) or a video (its frames decoded by cv2, through
    `VideoFlowRunner`).  Writes `<stem>_flow.png` (`%04d_flow.png` for a video), with `pred_bidir_flow` `_flow_bwd.png`,
    with `fwd_bwd_consistency_check` `_occ_fwd.png` / `_occ_bwd.png` (8-bit grey, occluded = 255) and with `save_flo_flow`
    `_pred.flo` (+ `_pred_bwd.flo`); `<stem>` is the first frame's name without its extension.  Pictures are coloured from
    the flow as written, resized and transposed back.

    `save_video` (a video only) writes `<video name>_flow.mp4` instead of the `_flow.png` pictures, or with
    `concat_flow_img` `<video name>_flow_img.mp4` of each pair's first frame and its picture side by side (stacked
    vertically for landscape frames), at the input's frame rate; the other files are written as without it.  The mp4 is
    encoded by cv2 with fourcc `mp4v` (MPEG-4 Part 2), not H.264 through imageio as the reference does, so its frames
    equal the pictures up to that codec's loss; an odd height or width is made even by repeating the last row or column.
    Unlike the reference, a pair is transposed back only when it is itself portrait (see the module docstring)."""
    if save_video and inference_video is None:
        raise ValueError("inference_flow: save_video needs inference_video")
    if fwd_bwd_consistency_check and not pred_bidir_flow:
        raise ValueError("inference_flow: fwd_bwd_consistency_check needs pred_bidir_flow=True")
    if (inference_dir is None) == (inference_video is None):
        raise ValueError("inference_flow needs one of inference_dir or inference_video")
    kw = dict(padding_factor=padding_factor, inference_size=inference_size, pred_bidir_flow=pred_bidir_flow,
              fwd_bwd_consistency_check=fwd_bwd_consistency_check, attn_type=attn_type, attn_splits_list=attn_splits_list,
              corr_radius_list=corr_radius_list, prop_radius_list=prop_radius_list, num_reg_refine=num_reg_refine)
    keys = flow_keys(pred_bidir_flow, fwd_bwd_consistency_check, save_flo_flow)
    return_flow = save_flo_flow or fwd_bwd_consistency_check
    rd = _Readers(readers, readers + 2 * batch)
    os.makedirs(output_path, exist_ok=True)
    if inference_video is not None:
        rd = _Readers(1, readers + 2 * batch)          # cv2 decodes a video frame after frame
        video = None
        if save_video:
            keys.remove("vis")
            video = (os.path.join(output_path, video_name(inference_video, concat_flow_img)), _video_fps(inference_video),
                     bool(concat_flow_img))
        return _video_flow(model, _video_frames(inference_video, rd), output_path, keys, return_flow, pred_bwd_flow, batch,
                           device, writers, kw, rd, video)
    files = flow_inputs(inference_dir)
    if len(files) < 2:
        return _stats({"pairs": 0, "steps": 0, "h2d_bytes": 0, "d2h_bytes": 0}, rd, 0.0)
    sizes = [_header_size(f) for f in files]
    alone = [t for t in range(len(files) - 1) if sizes[t] != sizes[t + 1]]
    for t in alone:
        ori = sizes[t][::-1] if sizes[t][0] > sizes[t][1] else sizes[t]
        if _inference_size(ori, padding_factor, inference_size) == ori:
            raise ValueError("inference_flow: %s and %s differ in size and the first needs no resize, so the model would "
                             "get frames of two sizes" % (files[t], files[t + 1]))
    cap = (max(h for h, _ in sizes), max(w for _, w in sizes))
    model.eval()
    runner = MixedSizeFlowRunner(model, cap, batch, device, pred_bwd_flow=pred_bwd_flow, visualize=True,
                                 return_flow=return_flow, max_buckets=max_buckets, **kw)
    names = _named(FLOW_FILES, keys, output_path, lambda t: flow_prefix(files, t, False))
    skip = set(alone)
    streamed = [t for t in range(len(files) - 1) if t not in skip]
    pairs = (p for t, p in enumerate(_consecutive(rd.map(_flow_frame, files))) if t not in skip)
    moved = {"h2d_bytes": 0, "d2h_bytes": 0}
    results = itertools.chain(((streamed[i], r) for i, r in runner.run(pairs)),
                              ((t, _flow_pair_alone(model, files[t], files[t + 1], device, pred_bwd_flow, kw, moved))
                               for t in alone))
    writer_s = _write_results(results, names, writers, batch)
    st = runner.stats
    return _stats({"pairs": st["pairs"] + len(alone), "steps": st["steps"] + len(alone),
                   "h2d_bytes": st["h2d_bytes"] + moved["h2d_bytes"], "d2h_bytes": st["d2h_bytes"] + moved["d2h_bytes"]},
                  rd, writer_s)


def _flow_pair_alone(model, file1, file2, device, pred_bwd_flow, kw, moved):
    """A pair whose two frames differ in size (a directory's size changes between them), taken as the reference takes
    it (evaluate_flow.py:710-760): both frames transposed when the first is portrait and resized from their own sizes to
    the first one's inference size, swapped with `pred_bwd_flow`, the flows brought back to the first frame's size.  The
    runners take pairs of one size, so such a pair runs alone through the same ops; its pictures are painted on the device."""
    kw = dict(kw)
    pf, size, bidir, check = (kw.pop(k) for k in ("padding_factor", "inference_size", "pred_bidir_flow",
                                                  "fwd_bwd_consistency_check"))
    frames = [_flow_frame(f) for f in (file1, file2)]
    x1, x2 = (torch.from_numpy(f).to(device).permute(2, 0, 1)[None].float() for f in frames)
    transposed = x1.shape[-2] > x1.shape[-1]
    if transposed:
        x1, x2 = x1.transpose(-2, -1), x2.transpose(-2, -1)
    ori = tuple(x1.shape[-2:])
    size = _inference_size(ori, pf, size)
    x1, x2 = _resize(x1, size), _resize(x2, size)
    if pred_bwd_flow:
        x1, x2 = x2, x1
    flow = model(x1, x2, pred_bidir_flow=bidir, task="flow", **kw)["flow_preds"][-1]
    out = _flow_outputs(flow, ori, size, transposed, bidir, check)
    out["vis"] = flow_to_image(out["flow"])
    if bidir:
        out["vis_bwd"] = flow_to_image(out["flow_bwd"])
    out = {k: v[0].cpu() for k, v in out.items()}
    moved["h2d_bytes"] += sum(f.nbytes for f in frames)
    moved["d2h_bytes"] += sum(v.numel() * v.element_size() for v in out.values())
    return out


def _video_fps(path):
    """CAP_PROP_FPS of the video, as utils/file_io.py:203-210 reads it; read before any device work, so that `save_video`
    on a video cv2 cannot open is refused at once"""
    import cv2
    cap = cv2.VideoCapture(path)
    try:
        if not cap.isOpened():
            raise ValueError("inference_flow: save_video cannot open the video %s to read its frame rate (cv2 reads it, and "
                             "cv2 with fourcc mp4v, not imageio as in the reference, writes the flow video)" % path)
        return cap.get(cv2.CAP_PROP_FPS)
    finally:
        cap.release()


def _video_flow(model, frames, output_path, keys, return_flow, pred_bwd_flow, batch, device, writers, kw, rd, video=None):
    """The video branch of `inference_flow` on a stream of RGB uint8 frames [H, W, 3] (all of one size); `video`: (path,
    fps, concat_flow_img) of the mp4 that `save_video` writes."""
    frames = iter(frames)
    first = next(frames, None)
    if first is None:
        return _stats({"pairs": 0, "steps": 0, "h2d_bytes": 0, "d2h_bytes": 0}, rd, 0.0)
    model.eval()
    concat = video is not None and video[2]
    runner = VideoFlowRunner(model, first.shape[:2], batch, device, visualize=True, return_flow=return_flow,
                             pred_bwd_flow=pred_bwd_flow, visualize_bwd=kw["pred_bidir_flow"], concat_frame=concat, **kw)
    names = _named(FLOW_FILES, keys, output_path, lambda t: flow_prefix(None, t, True))
    count = itertools.count()
    results = ((next(count), r) for r in runner.run(itertools.chain([first], frames)))
    writer = _VideoWriter(video[0], video[1], 2 * batch) if video is not None else None
    writer_s = _write_results(results, names, writers, batch, writer)
    return _stats(_sequence_stats(runner, next(count)), rd, writer_s)


@torch.no_grad()
def inference_stereo(model, inference_dir=None, inference_dir_left=None, inference_dir_right=None, output_path="output",
                     padding_factor=16, inference_size=None, attn_type=None, attn_splits_list=None, corr_radius_list=None,
                     prop_radius_list=None, num_reg_refine=1, pred_bidir_disp=False, pred_right_disp=False,
                     save_pfm_disp=False, batch=8, device="cuda", readers=4, writers=8, max_buckets=4):
    """`evaluate_stereo.inference_stereo`: the pairs of `inference_dir` (alternating files) or of `inference_dir_left` /
    `inference_dir_right`, decoded as `Image.open(f).convert('RGB')`, through `MixedSizeStereoRunner(visualize=True)`.
    Writes `<stem>_disp.png` (the `vis_disparity` picture, stored as cv2.imwrite stores it), with `save_pfm_disp`
    `<stem>_disp.pfm`, and with `pred_bidir_disp` the same for `<stem>_disp_right`; `<stem>` is the left file's name
    without its extension.  `pred_right_disp` writes the right view's disparity under the left names, as the reference."""
    if pred_bidir_disp and pred_right_disp:
        raise ValueError("inference_stereo: choose one of pred_bidir_disp / pred_right_disp")
    left, right = stereo_inputs(inference_dir, inference_dir_left, inference_dir_right)
    keys = stereo_keys(pred_bidir_disp, save_pfm_disp)
    rd = _Readers(readers, readers + 2 * batch)
    os.makedirs(output_path, exist_ok=True)
    if not left:
        return _stats({"pairs": 0, "steps": 0, "h2d_bytes": 0, "d2h_bytes": 0}, rd, 0.0)
    sizes = [_header_size(f) for f in left + right]
    cap = (max(h for h, _ in sizes), max(w for _, w in sizes))
    model.eval()
    runner = MixedSizeStereoRunner(model, cap, batch, device, padding_factor=padding_factor, inference_size=inference_size,
                                   pred_bidir_disp=pred_bidir_disp, pred_right_disp=pred_right_disp, visualize=True,
                                   return_disp=save_pfm_disp, max_buckets=max_buckets, attn_type=attn_type,
                                   attn_splits_list=attn_splits_list, corr_radius_list=corr_radius_list,
                                   prop_radius_list=prop_radius_list, num_reg_refine=num_reg_refine)
    names = _named(STEREO_FILES, keys, output_path, lambda i: _stem(left[i]))
    pairs = rd.map(lambda p: (_rgb_frame(p[0]), _rgb_frame(p[1])), zip(left, right))
    writer_s = _write_results(runner.run(pairs), names, writers, batch)
    st = runner.stats
    return _stats({k: st[k] for k in ("pairs", "steps", "h2d_bytes", "d2h_bytes")}, rd, writer_s)


@torch.no_grad()
def inference_depth(model, inference_dir=None, output_path="output", padding_factor=16, inference_size=None, attn_type="swin",
                    attn_splits_list=None, prop_radius_list=None, num_reg_refine=1, num_depth_candidates=64, min_depth=0.5,
                    max_depth=10, depth_from_argmax=False, pred_bidir_depth=False, batch=8, device="cuda", readers=4,
                    writers=8, max_buckets=4):
    """`evaluate_depth.inference_depth` on a ScanNet-layout directory: the consecutive pairs of color/*.jpg|png with the
    relative poses of pose/*.txt and the first intrinsic/*.txt (4x4, its [:3, :3]).  Writes `<stem>.png`, the
    `viz_depth_tensor(1 / depth)` picture, and with `pred_bidir_depth` `<stem>_bwd.png`; `<stem>` is the reference frame's
    name without its extension.  The intrinsics are not rescaled when the frames are resized, as in the reference.

    A directory of one frame size runs through `DepthSequenceRunner(visualize=True, return_depth=False)`, every frame
    encoded once.  Frames of several sizes run pair by pair through `MixedSizeDepthRunner` (`max_frame_size` from the
    image headers, at most `max_buckets` inference sizes holding graphs), as the reference takes each pair: both frames
    resized to the inference size of the first, the depth resized back to the first frame's size.  The reference resizes
    a pair only when its first frame is not already at the inference size (evaluate_depth.py:371-378), so a pair whose two
    frames differ in size while the first needs no resize would give its model frames of two sizes; such a directory is
    refused before any device work, as `inference_flow` refuses the same case."""
    if inference_dir is None:
        raise ValueError("inference_depth needs inference_dir")
    imgs, poses, intrinsics_file = depth_inputs(inference_dir)
    sizes = [_header_size(f) for f in imgs]
    for t in range(len(imgs) - 1):
        if sizes[t] != sizes[t + 1] and _inference_size(sizes[t], padding_factor, inference_size) == sizes[t]:
            raise ValueError("inference_depth: %s and %s differ in size and the first needs no resize, so the model would "
                             "get frames of two sizes" % (imgs[t], imgs[t + 1]))
    keys = depth_keys(pred_bidir_depth)
    rd = _Readers(readers, readers + 2 * batch)
    os.makedirs(output_path, exist_ok=True)
    if len(imgs) < 2:
        return _stats({"pairs": 0, "steps": 0, "h2d_bytes": 0, "d2h_bytes": 0}, rd, 0.0)
    model.eval()
    K = np.loadtxt(intrinsics_file).astype(np.float32).reshape((4, 4))[:3, :3]
    kw = dict(padding_factor=padding_factor, inference_size=inference_size, min_depth=min_depth, max_depth=max_depth,
              num_depth_candidates=num_depth_candidates, depth_from_argmax=depth_from_argmax,
              pred_bidir_depth=pred_bidir_depth, visualize=True, return_depth=False, attn_type=attn_type,
              attn_splits_list=attn_splits_list, prop_radius_list=prop_radius_list, num_reg_refine=num_reg_refine)
    names = _named(DEPTH_FILES, keys, output_path, lambda i: _stem(imgs[i]))
    items = rd.map(lambda p: (_rgb_frame(p[0]), _pose(p[1])), zip(imgs, poses))
    if len(set(sizes)) == 1:
        runner = DepthSequenceRunner(model, sizes[0], batch, device, K, **kw)
        writer_s = _write_results(enumerate(runner.run(items)), names, writers, batch)
        return _stats(_sequence_stats(runner, len(imgs) - 1, runner.pose_pin[0].nbytes), rd, writer_s)
    cap = (max(h for h, _ in sizes), max(w for _, w in sizes))
    runner = MixedSizeDepthRunner(model, cap, batch, device, K, max_buckets=max_buckets, **kw)
    pairs = ((a[0], b[0], _relative_poses([a[1], b[1]], False)[0]) for a, b in _consecutive(items))
    writer_s = _write_results(runner.run(pairs), names, writers, batch)
    st = runner.stats
    return _stats({k: st[k] for k in ("pairs", "steps", "h2d_bytes", "d2h_bytes")}, rd, writer_s)
