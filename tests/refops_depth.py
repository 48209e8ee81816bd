"""CPU statement of the depth-sequence op `frames_to_planar_normalized` (test infrastructure, like tests/refops.py and
tests/refops_video.py): the `-m gpu` tests compare the CUDA op with it, and `refops.register_cpu_kernels()` installs it as a
CPU kernel inside the test process, so the host logic of the depth sequence drivers runs on a machine without a GPU."""
import refops


def normalize_frames(frames, mean, std):
    """The depth pipeline's ToTensor + Normalize (dataloader/depth/augmentation.py:30, 56-61) on uint8 [T,H,W,3], on the CPU
    as the reference runs it: float32 planar frames, `/ 255.`, then per image and channel `sub_(mean).div_(std)`."""
    x = frames.permute(0, 3, 1, 2).float() / 255.
    for img in x:
        for t, m, s in zip(img, mean, std):
            t.sub_(m).div_(s)
    return x


def frames_to_planar_normalized(frames, h_out, w_out, mean, std):
    """uint8 [T,H,W,3] -> the normalised planar frames, resized (align_corners=True)."""
    return refops.resize_bilinear(normalize_frames(frames, mean, std).contiguous(), h_out, w_out, None, False)

