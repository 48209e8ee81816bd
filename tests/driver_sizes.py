"""The input sizes the drivers run the model at (the reference's submission and evaluation scripts and its datasets), next to
the bench resolutions of tests/test_stages_gpu.py.  Each size is derived with the drivers' own rule,
`unimatch_b200.inference._inference_size(raw, padding_factor, inference_size)`, from the dataset's raw frame size and the
script's flags; tests/test_driver_resolutions_cpu.py checks both the derivation and the model's divisibility rules.

At these sizes the 1/8 and 1/4 feature maps end on ragged query and key tiles that the bench sizes never reach, e.g.
352x1216: 6688 global-correlation tokens (last 128-row tile: 32 rows), 1/8 windows of 1672 tokens (tail 8), 1/4 windows of
418 (tail 34)."""
from collections import namedtuple

# raw: the dataset's frame size (None: frames of any size are resized to inference_size)
Case = namedtuple("Case", "workload H W bidir raw padding inference_size origin")

SINTEL = (436, 1024)
KITTI = (375, 1242)

CASES = [
    Case("gmflow-scale2-regrefine6", 416, 1024, False, SINTEL, 32, (416, 1024),
         "Sintel submission: scripts/gmflow_submission.sh, --inference_size 416 1024 --padding_factor 32"),
    Case("gmflow-scale2-regrefine6", 352, 1216, False, KITTI, 32, (352, 1216),
         "KITTI flow submission: scripts/gmflow_submission.sh, --inference_size 352 1216 --padding_factor 32"),
    Case("gmflow-scale2-regrefine6", 384, 1248, False, KITTI, 32, None,
         "KITTI flow validation: scripts/gmflow_evaluate.sh, --padding_factor 32 (kitti-mode padding of 375x1242)"),
    Case("gmflow-scale2-regrefine6", 352, 1216, True, KITTI, 32, (352, 1216),
         "KITTI flow submission size with --pred_bidir_flow (scripts/gmflow_demo.sh)"),
    Case("gmflow-scale1", 448, 1024, False, SINTEL, 16, None,
         "Sintel validation: scripts/gmflow_evaluate.sh, gmflow-scale1 with the default --padding_factor 16"),
    Case("gmstereo-scale2-regrefine3", 352, 1216, False, KITTI, 32, (352, 1216),
         "KITTI 2015 stereo submission: scripts/gmstereo_submission.sh, --inference_size 352 1216"),
    Case("gmstereo-scale2-regrefine3", 1024, 1536, False, None, 32, (1024, 1536),
         "Middlebury submission: scripts/gmstereo_submission.sh, --inference_size 1024 1536 (frames of any size resized)"),
    Case("gmstereo-scale2-regrefine3", 512, 768, False, None, 32, (512, 768),
         "ETH3D submission: scripts/gmstereo_submission.sh, --inference_size 512 768 (frames of any size resized)"),
    Case("gmstereo-scale2", 384, 1248, False, KITTI, 32, None,
         "KITTI 2015 stereo validation: scripts/gmstereo_evaluate.sh, --padding_factor 32, no inference size"),
    Case("gmdepth-scale1", 480, 640, False, (480, 640), 16, None,
         "depth evaluation: the reference's depth loader resizes every frame to 640x480, default --padding_factor 16"),
    Case("gmdepth-scale1-regrefine1", 480, 640, False, (480, 640), 16, None,
         "depth evaluation: scripts/gmdepth_evaluate.sh, 640x480 frames"),
    Case("gmdepth-scale1-regrefine1", 480, 640, True, (480, 640), 16, None,
         "640x480 depth frames with --pred_bidir_depth (scripts/gmdepth_demo.sh)"),
]


def case_id(c):
    return "%s-%dx%d%s" % (c.workload, c.H, c.W, "-bidir" if c.bidir else "")
