"""CPU: the MViT builder variants (tests/golden/mvit_variants.pt, oracle/gen_golden_mvit_variants.py) - module trees,
fuse_bn(), the deprecation warning, the host-side plans and the pre-activation prologue fields of pv_conv3d_desc."""
import ctypes
import os
import subprocess
import tempfile
import warnings

import pytest
import torch

import pytorchvideo_b200.layers.attention as PA
import pytorchvideo_b200.models.vision_transformers as PV
from pytorchvideo_b200 import testing as TS
from pytorchvideo_b200.engine.lower import lower_only

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CASES = sorted(TS.MVIT_VARIANT_CASES)
LN_OPS = (".norm1", ".norm2", ".norm", ".add", "norm_embed")       # the LayerNorm launches of an MViT plan


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(HERE, "golden", "mvit_variants.pt"), weights_only=False)


def _build(case, **kw):
    return TS.build_mvit_variant_case(case, PV.create_multiscale_vision_transformers, PA.MultiScaleBlock, **kw)


def _plan(case, dtype="f16"):
    model, x, extra = _build(case)
    plan, shape = lower_only(model, torch.zeros(x.shape), dtype=dtype, extra=tuple(tuple(e) for e in extra))
    return plan, shape, [m["name"] for m in plan.meta]


@pytest.mark.parametrize("case", CASES)
def test_module_tree_matches_the_reference(gold, case):
    """state_dict keys, shapes, values and repr equal the reference's, before fuse_bn() and after it."""
    g = gold[case]
    model, x, _ = _build(case)
    sd = model.state_dict()
    assert list(sd.keys()) == g["keys"]
    assert [list(v.shape) for v in sd.values()] == g["shapes"]
    assert repr(model) == g["repr"]
    assert abs(TS.state_checksum(model) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"])
    assert TS.tensor_checksum(x) == pytest.approx(g["input_checksum"], rel=1e-9)
    assert sum(isinstance(m, (torch.nn.BatchNorm1d, torch.nn.BatchNorm3d)) for m in model.modules()) == g["batchnorms"]


@pytest.mark.parametrize("case", CASES)
def test_reference_tree_lowers_to_the_same_plan(gold, case):
    """The lowering dispatches on module classes and attributes: this package's tree and the reference's give one plan."""
    plan, shape, _ = _plan(case)
    assert [n for n, _ in plan.ops] == gold[case]["ref_ops"]
    assert dict(plan.stats) == gold[case]["ref_stats"]
    assert list(shape) == gold[case]["out_shape"] == list(gold[case]["output"].shape)


def test_fuse_bn_keeps_the_attention_pool_batchnorms():
    """fuse_bn() folds norm1 / norm2 and replaces attn.norm_{q,k,v}, but the _attention_pool wrappers still hold the
    BatchNorm3d modules that forward applies (as in the reference)."""
    model, _, _ = _build("bn_mvit_b_fused")
    blk = model.blocks[1]
    assert type(blk.norm1).__name__ == type(blk.norm2).__name__ == "Identity" and blk.norm1_is_batchnorm_1d
    assert type(blk.attn.norm_q).__name__ == "Identity"
    assert isinstance(blk.attn._attention_pool_q.norm, torch.nn.BatchNorm3d)
    assert sum(isinstance(m, (torch.nn.BatchNorm1d, torch.nn.BatchNorm3d)) for m in model.modules()) == 35


def test_scriptable_batchnorm_model_warns(gold):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        PV.create_multiscale_vision_transformers(spatial_size=32, temporal_size=2, depth=1, norm="batchnorm",
                                                 create_scriptable_model=True)
    got = [(c.category.__name__, str(c.message)) for c in w if issubclass(c.category, DeprecationWarning)]
    assert got == gold["_scriptable_warning"] and len(got) == 1
    with warnings.catch_warnings(record=True) as w:      # layernorm + create_scriptable_model keeps its behaviour
        warnings.simplefilter("always")
        PV.create_multiscale_vision_transformers(spatial_size=32, temporal_size=2, depth=1, create_scriptable_model=True)
    assert not [c for c in w if issubclass(c.category, DeprecationWarning)]


@pytest.mark.parametrize("case", ["bn_mvit_b", "bn_mvit_b_fused", "bn_small"])
def test_batchnorm_mvit_plan_has_no_layernorm_and_one_kv_pool_per_block(case):
    """BatchNorm1d block norms fold into the linears (no launch), the attention-pool BatchNorm3d + GELU is the depthwise
    prologue (no norm launch), and K | V pool in one launch per block."""
    model, _, _ = _build(case)
    for dtype in ("f16", "f32"):
        plan, _, names = _plan(case, dtype)
        assert not plan.trunk32
        assert not [n for n in names if n.endswith(LN_OPS)], [n for n in names if n.endswith(LN_OPS)]
        kv = sum(b.attn.pool_k is not None for b in model.blocks)
        assert sum(n.endswith(".pool_kv.dwconv") for n in names) == kv > 0
        assert not [n for n in names if ".pool_k." in n or ".pool_v." in n]
        q = sum(b.attn.pool_q is not None for b in model.blocks)
        assert plan.stats["pool_prologue"] == kv + q


def test_pool_first_batchnorm_materialises_x_norm_once_per_block():
    model, _, _ = _build("pool_first_bn")
    for dtype in ("f16", "f32"):
        _, _, names = _plan("pool_first_bn", dtype)
        assert [n for n in names if n.endswith(".norm1")] == ["blocks.%d.norm1" % i for i in range(len(model.blocks))]
        assert not [n for n in names if n.endswith((".norm2", ".norm", "norm_embed"))]


def test_variant_plans_on_the_host():
    _, shape, names = _plan("head_none")
    assert shape == (2, 33, 384) and not [n for n in names if n.startswith("head")]
    for case in ("tokens", "tokens_no_cls"):
        _, shape, names = _plan(case)
        assert shape == (2, 400) and not [n for n in names if n.startswith("patch_embed")]
    _, _, names = _plan("avg")
    assert sum(n.endswith(".avgpool") for n in names) == 8 and not [n for n in names if n.endswith(".dwconv")]
    _, _, names = _plan("pool_first_ln")
    assert sum(n.endswith((".attn.q", ".attn.k", ".attn.v")) for n in names) == 12


@pytest.mark.parametrize("case", ["tokens", "tokens_no_cls"])
def test_token_input_must_match_the_patch_grid(case):
    model, _, _ = _build(case)
    with pytest.raises(RuntimeError):
        lower_only(model, torch.zeros(2, 4 * 28 * 28 - 1, 96))
    with pytest.raises(RuntimeError):
        lower_only(model, torch.zeros(2, 4 * 28 * 28, 88))


def test_full_pooling_convs_still_raise():
    model = PV.create_multiscale_vision_transformers(spatial_size=64, temporal_size=4, depth=2, depthwise_conv=False,
                                                     pool_q_stride_size=[[1, 1, 2, 2]]).eval()
    with pytest.raises(NotImplementedError):
        lower_only(model, torch.zeros(1, 3, 4, 64, 64))


def test_prologue_fields_match_the_header():
    """The ctypes mirror puts pre_scale / pre_bias / pre_act where the C header does (gcc offsetof probe)."""
    from pytorchvideo_b200 import _lib
    probe = r'''
    #include <stddef.h>
    #include <stdio.h>
    #include "pv_b200.h"
    int main(){ printf("%zu %zu %zu %zu\n", offsetof(pv_conv3d_desc, pre_scale), offsetof(pv_conv3d_desc, pre_bias),
                       offsetof(pv_conv3d_desc, pre_act), sizeof(pv_conv3d_desc)); return 0; }'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "p.c")
        open(c, "w").write(probe)
        exe = os.path.join(td, "p")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True).stdout.split()]
    D = _lib.Conv3dDesc
    assert got == [D.pre_scale.offset, D.pre_bias.offset, D.pre_act.offset, ctypes.sizeof(D)]
    assert (D().pre_scale, D().pre_bias, D().pre_act) == (None, None, 0)     # zero-initialised: no prologue
