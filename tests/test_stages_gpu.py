"""Parity where the metric lives: `unimatch_b200.UniMatch` on the GPU against the oracle (== reference) at the BASELINE
shape -- one 480x832 pair, gmflow-scale2-regrefine6 -- stage by stage with teacher forcing (every stage fed the oracle's
inputs for it, so errors neither hide nor compound; reference unimatch/unimatch.py:136-354), then free-running end to end.
The oracle runs on the box's CPU (~15-30 s).  Tolerances: tests/stage_checks.py."""
import pytest
import torch

import stage_checks

pytestmark = pytest.mark.gpu


def test_teacher_forced_stages_480x832_regrefine6():
    lines = []
    try:
        stage_checks.run(torch.device("cuda", 0), report=lines.append)
    finally:
        print("\n".join(lines))
