"""CPU statement of the stereo op `disparity_to_image` (test infrastructure, like tests/refops.py and tests/refops_video.py):
the `-m gpu` tests compare the CUDA op with it, and `refops.register_cpu_kernels()` installs it as a CPU kernel inside the
test process, so the host logic of the stereo drivers runs on a machine without a GPU."""
import torch

from oracle import disp_viz as OD


def disparity_to_image(disp, out):
    out.copy_(torch.from_numpy(OD.vis_disparity_batch(disp.detach().cpu().numpy())))

