"""Parity where the metric lives: `unimatch_b200.UniMatch` on the GPU against the oracle (== reference), one pair of every
workload at its bench resolution -- flow 480x832, stereo 544x960, depth 384x512 -- plus gmflow-scale2-regrefine6 with
pred_bidir_flow and gmdepth-scale1-regrefine1 with pred_bidir_depth, also at the bench resolution.  Stage by stage with teacher
forcing (every stage fed the oracle's inputs for it, so errors neither hide nor compound; reference unimatch/unimatch.py:136-354),
then free-running end to end.  The oracle runs on the host's CPU; its forward took, with 8 CPU threads: gmflow-scale1 1.6 s,
gmflow-scale2 4.8 s, gmflow-scale2-regrefine6 14 s (bidirectional 24 s), gmstereo-scale2 4.4 s, gmstereo-scale2-regrefine3
9.4 s, gmdepth-scale1 0.4 s, gmdepth-scale1-regrefine1 0.5 s (bidirectional 0.8 s).  Tolerances: tests/stage_checks.py."""
import pytest
import torch

import stage_checks
from unimatch_b200.spec import WORKLOADS

pytestmark = pytest.mark.gpu


def run_bench_resolution(workload, bidir):
    H, W = stage_checks.BENCH_HW[WORKLOADS[workload]["model"]["task"]]
    lines = []
    try:
        stage_checks.run(torch.device("cuda", 0), workload, H, W, bidir, report=lines.append)
    finally:
        print("\n" + "\n".join(lines))


def test_teacher_forced_stages_480x832_regrefine6():
    run_bench_resolution("gmflow-scale2-regrefine6", False)


@pytest.mark.parametrize("workload,bidir", [c for c in stage_checks.CASES if c != ("gmflow-scale2-regrefine6", False)])
def test_teacher_forced_stages_at_bench_resolution(workload, bidir):
    run_bench_resolution(workload, bidir)
