"""The batch audit (test_gpu_batch_audit.py) on the audio, efficient, MViT-variant and masked cases in f16, and every f32 row but the SSL trunks: each row's launches against float64 on every clip, and
each clip's bits invariant under reordering the batch and against the batch-1 plan."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from test_gpu_batch_audit import run_row  # noqa: E402

SWEEP = [r for r in TS.batch_sweep(bench.WORKLOADS) if TS.batch_sweep_part(r, bench.WORKLOADS) == "layers"]


@pytest.mark.gpu
@pytest.mark.parametrize("prec,family,case,B,checks", SWEEP, ids=["%s-%s-%s-b%d" % r[:4] for r in SWEEP])
def test_batch_audit(prec, family, case, B, checks):
    run_row(prec, family, case, B, checks)
