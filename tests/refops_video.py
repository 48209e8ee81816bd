"""CPU statements of the video ops `frames_to_planar` and `flow_to_image` (test infrastructure, like tests/refops.py):
the `-m gpu` tests compare the CUDA ops with these, and `refops.register_cpu_kernels()` installs them as CPU kernels inside
the test process, so the host logic of the video drivers runs on a machine without a GPU."""
import torch

import refops
from oracle import flow_viz as OV


def frames_to_planar(frames, h_out, w_out, transpose):
    """uint8 [T,H,W,3] -> the planar float frames, transposed to [T,3,W,H] when asked, resized (align_corners=True)."""
    x = frames.permute(0, 3, 1, 2).float()
    if transpose:
        x = x.transpose(-2, -1)
    return refops.resize_bilinear(x.contiguous(), h_out, w_out, None, False)


def flow_to_image(flow, out):
    out.copy_(torch.from_numpy(OV.flow_to_image_batch(flow.detach().cpu().numpy())))

