"""CPU statement of the stereo op `disparity_to_image` (test infrastructure, like tests/refops.py and tests/refops_video.py):
the `-m gpu` tests compare the CUDA op with it, and `register_cpu_kernels()` installs it -- together with every op of
refops.py, refops_video.py and refops_depth.py -- as a CPU kernel inside the test process, so the host logic of the stereo
drivers runs on a machine without a GPU."""
import torch

import refops_depth
from oracle import disp_viz as OD


def disparity_to_image(disp, out):
    out.copy_(torch.from_numpy(OD.vis_disparity_batch(disp.detach().cpu().numpy())))


ALL = ["disparity_to_image"]

_registered = []


def register_cpu_kernels():
    refops_depth.register_cpu_kernels()
    if _registered:
        return
    lib = torch.library.Library("unimatch_sm100", "IMPL", "CPU")
    g = globals()
    for name in ALL:
        lib.impl(name, g[name])
    _registered.append(lib)
