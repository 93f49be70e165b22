"""CPU: the image MViT-B-16 and SlowFast-16x8-R101-50-50 hub entries - module trees, host lowering, plane-kernel
routing and the error paths.  tests/golden/hub_tail.pt (oracle/gen_golden_hub.py) holds what the reference built."""
import ctypes
import os
import re

import pytest
import torch

import pytorchvideo_b200.models.hub as PH
from pytorchvideo_b200 import _lib as L
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.engine.lower import lower_only

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "pytorchvideo_b200", "csrc")


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(HERE, "golden", "hub_tail.pt"), weights_only=False)


def _zeros(case):
    B, shape = TS.HUB_TAIL_CASES[case]
    if len(shape) == 3:
        return torch.zeros(B, *shape)
    return TS.slowfast_inputs(torch.zeros(B, *shape))


@pytest.mark.parametrize("case", sorted(TS.HUB_TAIL_CASES))
def test_builders_match_the_reference_tree(gold, case):
    m = getattr(PH, case)()
    sd = m.state_dict()
    assert list(sd.keys()) == gold[case]["keys"]
    assert [list(v.shape) for v in sd.values()] == gold[case]["shapes"]
    assert repr(m) == gold[case]["repr"]


@pytest.mark.parametrize("case", sorted(TS.HUB_TAIL_CASES))
def test_pretrained_weights_are_refused(case):
    with pytest.raises(RuntimeError, match="download"):
        getattr(PH, case)(pretrained=True)


@pytest.mark.parametrize("case", sorted(TS.HUB_TAIL_CASES))
def test_lowering_matches_the_reference_tree(gold, case):
    """(B, 400) logits, and the same op sequence and kernel counts as the plan of the reference's own module tree."""
    plan, shape = lower_only(getattr(PH, case)().eval(), _zeros(case))
    assert list(shape) == [TS.HUB_TAIL_CASES[case][0], 400] == gold[case]["out_shape"]
    assert [n for n, _ in plan.ops] == gold[case]["ref_ops"]
    assert plan.stats == gold[case]["ref_stats"]


def test_image_mvit_dry_run_counts_match_the_reference_macs(gold):
    plan, shape = lower_only(PH.mvit_base_16().eval(), torch.zeros(1, 3, 224, 224))
    assert tuple(shape) == (1, 400)
    macs = sum(x["flops"] for x in plan.meta) / 2
    assert abs(macs - gold["mvit_base_16"]["ref_macs_per_image"]) <= 1e-6 * macs
    assert abs(macs / 1e9 - 7.809) < 0.001


def test_image_mvit_routes():
    """The 7x7 / stride 4 embed reads the W-padded image on the tensor cores (window mode); all 19 attention pools
    (3 pool_q, 16 fused K|V) run on the plane kernel; the skip max-pools keep pv_pool3d_fwd."""
    plan, _ = lower_only(PH.mvit_base_16().eval(), torch.zeros(4, 3, 224, 224))
    kinds = {md["name"]: md["kind"] for md in plan.meta}
    assert plan.meta[0]["name"] == "ncdhw_to_ndhwc_padw"
    assert kinds["patch_embed.patch_model"] == "tcgen05"
    pools = [n for n in kinds if n.endswith(".dwconv")]
    assert len(pools) == 19 and sum(n.endswith("pool_q.dwconv") for n in pools) == 3
    assert plan.stats["dwplane"] == 19
    assert sum(n.endswith(".maxpool") for n in kinds) == 3


def test_video_mvit_keeps_its_pool_routes():
    plan, _ = lower_only(PH.mvit_base_16x4().eval(), torch.zeros(1, 3, 16, 224, 224))
    assert "dwplane" not in plan.stats


def test_slowfast_16x8_fast_pathway_routes():
    """64 Fast frames: the Fast res2 / res3 blocks stay fused, the stems keep their tensor-core routes."""
    plan, _ = lower_only(PH.slowfast_16x8_r101_50_50().eval(), TS.slowfast_inputs(torch.zeros(8, 3, 64, 224, 224)))
    assert plan.stats["fused_block"] == 7
    assert plan.stats.get("stem_stream", 0) + plan.stats.get("stem_rows", 0) == 2
    assert plan.stats["direct"] == 0


def test_four_d_input_to_a_video_model_raises():
    for m, x in ((PH.x3d_xs().eval(), torch.zeros(1, 3, 160, 160)), (PH.mvit_base_16x4().eval(), torch.zeros(1, 3, 224, 224))):
        with pytest.raises(RuntimeError, match="image MViT"):
            lower_only(m, x)


def test_image_mvit_refuses_a_clip():
    with pytest.raises(RuntimeError, match="images"):
        lower_only(PH.mvit_base_16().eval(), torch.zeros(1, 3, 1, 224, 224))


def test_2d_patch_needs_one_frame():
    from pytorchvideo_b200.models.vision_transformers import create_multiscale_vision_transformers
    with pytest.raises(AssertionError, match="temporal_size"):
        create_multiscale_vision_transformers(spatial_size=224, temporal_size=2, use_2d_patch=True,
                                              conv_patch_embed_kernel=(7, 7), conv_patch_embed_stride=(4, 4),
                                              conv_patch_embed_padding=(3, 3))


def _plane_desc(H, W, C, s, N=2, dtype=L.PV_F16, kt=1, T=1, row_stride=None, batch_stride=None):
    d = L.Conv3dDesc()
    d.dtype, d.N, d.Ti, d.Hi, d.Wi, d.Ci = dtype, N, T, H, W, C
    d.To, d.Ho, d.Wo, d.Co = T, (H + 2 - 3) // s + 1, (W + 2 - 3) // s + 1, C
    d.kt, d.kh, d.kw = kt, 3, 3
    d.st, d.sh, d.sw = 1, s, s
    d.pt, d.ph, d.pw = (kt - 1) // 2, 1, 1
    d.dt, d.dh, d.dw = 1, 1, 1
    d.groups = C
    d.x_row_stride = row_stride or C
    d.y_row_stride = C
    d.x_batch_stride = batch_stride if batch_stride is not None else (1 + H * W) * d.x_row_stride
    return d


def test_plane_probe_answers_for_the_image_pools_only():
    lib = L.load()
    ok = lambda d: lib.pv_dwplane_supported(ctypes.byref(d))      # noqa: E731
    for s in (1, 2, 4):
        for H in (56, 28, 14, 7):
            assert ok(_plane_desc(H, H, 96, s)) == 1
    assert ok(_plane_desc(56, 56, 1536, 4, row_stride=2304)) == 1
    assert ok(_plane_desc(14, 14, 96, 3)) == 0                       # stride 3
    assert ok(_plane_desc(14, 14, 96, 1, dtype=L.PV_F32)) == 0       # f32 storage
    assert ok(_plane_desc(14, 14, 96, 1, kt=3, T=4)) == 0            # a video pool
    assert ok(_plane_desc(14, 14, 92, 1)) == 0                       # channels not a multiple of 8
    assert ok(_plane_desc(14, 14, 96, 1, batch_stride=197 * 96 + 4)) == 0


PLANE_INSTANCES = {"dwconv_plane_kernel<%s,%s,%s>" % (s, ph, pw) for s in (1, 2) for ph, pw in ((4, 4), (2, 7))} | \
    {"dwconv_plane_kernel<4,1,2>"}


def test_plane_instance_ledger():
    src = open(os.path.join(CSRC, "pv_dwplane.cu")).read()
    compiled = {"dwconv_plane_kernel<%s,%s,%s>" % a for a in re.findall(r"PV_DWP\((\d+), (\d+), (\d+)\);", src)}
    assert compiled == PLANE_INSTANCES
    assert '"dwconv_plane_kernel<" #S_ "," #PH_ "," #PW_ ">"' in src
