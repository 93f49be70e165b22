"""The launch footprint walk and the legal-order runs (test_gpu_launch_footprint.py) on the f32 parity-mode plans of
every audit_catalogue case, and of the multi-lane cases at batch 3."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from test_gpu_launch_footprint import run_row  # noqa: E402

CASES = [r for r in TS.footprint_cases(bench.WORKLOADS) if TS.footprint_part(r) == "f32"]


@pytest.mark.gpu
@pytest.mark.parametrize("prec,family,case,batch", CASES, ids=["%s-%s-%s-b%s" % r for r in CASES])
def test_launch_footprint(prec, family, case, batch):
    run_row(prec, family, case, batch)
