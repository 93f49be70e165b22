"""GPU: end-to-end model parity.  CUDA engine vs (a) golden logits produced by the REAL reference
(tests/golden/model_*.pt) and (b) the oracle re-run on this box.

Tolerances (also in DESIGN.md):
  f32 storage ("parity mode", CUDA-core kernels): |d| <= 1e-3*|ref| + 1e-4*max(1, max|ref|)
      i.e. the north-star rtol=1e-3 / atol=1e-4 with atol expressed relative to the logit scale
      (synthetic weights give logits of magnitude 10..500).
  f16 storage (tensor-core path, the benchmarked one): per-case MEASURED bounds are asserted - the
      fraction of logits inside rtol=1e-3/atol=1e-4*scale and max|d|/max|ref| (F16_BOUNDS below).
"""
import os

import pytest
import torch

from oracle.interp import oracle_forward
from pytorchvideo_b200 import testing as TS
import pytorchvideo_b200.models.hub as PH

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _to_dev(inp):
    return [t.cuda() for t in inp] if isinstance(inp, list) else inp.cuda()


@pytest.mark.parametrize("case", ["x3d_xs", "x3d_m", "slowfast_r50", "slow_r50", "csn_r101", "r2plus1d_r50", "i3d_r50",
                                  "mvit_base_8x112", "mvit_base_16x4", "c2d_r50", "x3d_s", "c1_x3d_xs"])
def test_model_f32_parity_mode(case):
    from pytorchvideo_b200 import config
    g, model, inp, _ = _setup_case(case)
    ref = g["output"]
    config.set_precision("f32")
    try:
        model.cuda()
        out = model(_to_dev(inp)).float().cpu()
    finally:
        config.set_precision("f16")
        model.cpu()
    scale = max(1.0, float(ref.abs().max()))
    err = (out - ref).abs()
    tol = 1e-3 * ref.abs() + 1e-4 * scale
    assert out.shape == ref.shape
    assert bool((err <= tol).all()), "max err %.3e (scale %.3g)" % (float(err.max()), scale)


# ---- f16 tensor-core path (the benchmarked configuration) -------------------------------------------------
# Asserted per case: (minimum fraction of logits inside rtol 1e-3 / atol 1e-4*max(1,max|ref|), maximum
# max|d|/max|ref|).  The numbers are measured values with a small margin (they hold on H100), so a numerical
# regression fails the suite; they are not aspirations.
#  * arbitrary fp32 weights: rounding the WEIGHTS to f16 operands alone moves 8-25 % of the logits out of
#    the band even in the reference's own fp32 arithmetic (tests/test_oracle_pinning.py::
#    test_f16_operand_floor_of_the_reference_arithmetic) - no f16-operand tensor-core path can do better;
#  * "f16 grid" cases (weights and clip exactly representable in f16, so reference and engine multiply
#    IDENTICAL operands, BASELINE batch sizes): what is left is activation rounding + summation order.
F16_BOUNDS = {
    # case: (min in-band fraction, max |d|/max|ref|)
    "x3d_xs": (0.78, 1.0e-3),
    "x3d_s": (0.70, 1.1e-3),
    "x3d_m": (0.73, 1.2e-3),
    "x3d_l": (0.65, 1.5e-3),
    "slowfast_r50": (0.85, 9e-4),
    "slowfast_r101": (0.84, 1.0e-3),
    "slow_r50": (0.83, 1.1e-3),
    "c2d_r50": (0.82, 8e-4),
    "csn_r101": (0.84, 8e-4),
    "i3d_r50": (0.83, 9e-4),
    # MViT: fp32 residual trunk (pv_add_layernorm)
    "mvit_base_8x112": (0.61, 1.6e-3),
    "mvit_base_16x4": (0.67, 1.2e-3),
    "mvit_base_32x3": (0.64, 1.3e-3),
    # softmax head: the outputs are probabilities, |d p| ~ p * |d logit| - the relative error of the largest
    # probability is the ABSOLUTE logit error (~5e-4 * |logit| scale 15)
    "r2plus1d_r50": (0.97, 1.2e-2),
    # f16-grid weights / inputs (identical operands), BASELINE configs at their real batch sizes
    "c1_x3d_xs": (0.94, 7e-4),
    "c2_slowfast_r50_b8": (0.96, 7e-4),
    "c3_mvit_base_16x4_b8": (0.84, 9e-4),
    "c4_x3d_m_b32": (0.92, 9e-4),
    "slow_r50_f16w": (0.96, 8e-4),
    "mvit_base_8x112_f16w": (0.79, 1.1e-3),
}
_BIG = ("c2_slowfast_r50_b8", "c3_mvit_base_16x4_b8", "c4_x3d_m_b32", "x3d_l", "mvit_base_32x3", "slowfast_r101")


def _setup_case(case):
    g = torch.load(os.path.join(GOLD, "model_%s.pt" % case), weights_only=False)
    model, inp, is_sf = TS.build_case(case, PH, weight_seed=g["weight_seed"], input_seed=g["input_seed"])
    assert abs(TS.state_checksum(model) - g["state_checksum"]) <= 1e-6 * abs(g["state_checksum"]), "weights differ from the golden's"
    return g, model, inp, is_sf


@pytest.mark.parametrize("case", sorted(F16_BOUNDS))
def test_model_f16_tensor_core_path(case):
    g, model, inp, _ = _setup_case(case)
    ref = g["output"]
    model.cuda()
    out = model(_to_dev(inp)).float().cpu()
    out2 = model(_to_dev(inp)).float().cpu()           # cached plan + graph replay is deterministic
    model.cpu()
    assert torch.equal(out, out2)       # SE channel sums are integer (fixed-point) atomics: order-independent
    assert out.shape == ref.shape
    scale = float(ref.abs().max())
    err = (out - ref).abs()
    inside = float((err <= 1e-3 * ref.abs() + 1e-4 * max(1.0, scale)).float().mean())
    rel = float(err.max()) / scale
    print("PARITY %s f16: max|d|/max|ref| = %.3e, fraction within rtol1e-3/atol1e-4 = %.3f" % (case, rel, inside))
    lo, hi = F16_BOUNDS[case]
    assert rel <= hi, "max|d|/max|ref| = %.3e > %.1e" % (rel, hi)
    if lo is not None:
        assert inside >= lo, "only %.3f of the logits inside the band (floor %.2f)" % (inside, lo)
    if case not in _BIG:
        # the oracle re-run here agrees with the golden (same arithmetic, this box's CPU)
        orc = oracle_forward(model, inp)
        assert float((orc - ref).abs().max()) <= 1e-4 * max(1.0, scale)


def test_batch_shards_are_independent():
    """Eval forward has no cross-sample coupling: f(batch)[i] == f(batch[i:i+1]) (what makes the
    multi-GPU sharding collective-free)."""
    model = TS.randomize_model(PH.x3d_xs(), seed=7).eval().cuda()
    clip = TS.synthetic_clip(3, 4, 160, 160, seed=3).cuda()
    full = model(clip).cpu()
    for i in range(3):
        one = model(clip[i:i + 1]).cpu()
        assert torch.allclose(one, full[i:i + 1], rtol=1e-3, atol=1e-3 * float(full.abs().max()))


def test_wrong_channels_raise_runtimeerror_on_gpu():
    model = PH.x3d_xs().eval().cuda()
    with pytest.raises(RuntimeError):
        model(torch.zeros(1, 4, 4, 160, 160, device="cuda"))


def test_pipelined_serving_matches_direct_call():
    """engine/pipeline.py: double-buffered host-in/host-out loop returns, in order, exactly what the
    plain call returns for every batch (copies overlap compute; results must not be mixed up)."""
    from pytorchvideo_b200.engine.lower import compile_model
    model = TS.randomize_model(PH.slow_r50(), seed=11).eval()
    batches = [TS.synthetic_clip(1, 8, 224, 224, seed=20 + i).pin_memory() for i in range(5)]
    cm = compile_model(model, batches[0].cuda(), dtype="f16")
    direct = [cm(b.cuda()).float().cpu().clone() for b in batches]
    assert not torch.equal(direct[0], direct[1])
    pipe = cm.pipeline(depth=2)
    got = list(pipe.run(batches))
    assert len(got) == len(batches)
    for g, d in zip(got, direct):
        assert torch.equal(g, d)
    t = pipe.submit(batches[3])
    assert torch.equal(pipe.result(t), direct[3])
    with pytest.raises(RuntimeError):
        pipe.result(t + 1)


def test_full_size_bench_config_properties():
    """BASELINE configs[1] at FULL size (SlowFast-8x8-R50, 8 clips of 3x32x224x224): too big for the CPU oracle
    in a test, so check size-independent properties of the eval forward instead: per-sample independence
    (what makes the multi-GPU sharding collective-free), batch-permutation equivariance and determinism."""
    model = TS.randomize_model(PH.slowfast_r50(), seed=5).eval().cuda()
    clip = TS.synthetic_clip(8, 32, 224, 224, seed=9)
    inp = [t.cuda() for t in TS.slowfast_inputs(clip)]
    full = model(inp).float().cpu().clone()
    assert full.shape == (8, 400) and bool(torch.isfinite(full).all())
    again = model(inp).float().cpu()
    assert torch.equal(full, again)                       # tensor-core path is deterministic
    scale = float(full.abs().max())
    for i in (0, 7):
        one = model([t[i:i + 1] for t in inp]).float().cpu()
        assert torch.allclose(one, full[i:i + 1], rtol=1e-3, atol=1e-3 * scale), float((one - full[i:i + 1]).abs().max())
    perm = torch.tensor([3, 0, 7, 1, 6, 2, 5, 4])
    permuted = model([t[perm.to(t.device)] for t in inp]).float().cpu()
    assert torch.allclose(permuted, full[perm], rtol=1e-3, atol=1e-3 * scale)


def test_accelerator_transmute_route_matches_golden():
    """The reference's plug-in protocol (accelerator/deployment/common/model_transmuter.py:53-86 +
    mobile_cpu/utils/model_conversion.py:87-125) with target "b200": every top-level block of a model is replaced
    by a B200Block, each block is converted with the input size recorded by one hooked forward, and the converted
    model reproduces the reference golden like the whole-tree plan does (f16 tolerances of F16_BOUNDS)."""
    from pytorchvideo_b200.accelerator import B200Block, convert_to_deployable_form, transmute_model
    g, model, inp, _ = _setup_case("c1_x3d_xs")
    model.cuda()
    x = inp.cuda()
    whole = model(x).float().cpu()
    one = convert_to_deployable_form(model, x)                 # untouched model the engine lowers whole: ONE block
    assert isinstance(one, B200Block) and one._compiled is not None
    assert float((one(x).float().cpu() - whole).abs().max()) <= 1e-3 * float(whole.abs().max())   # same plan
    dep = convert_to_deployable_form(model, x, whole_model=False)
    blocks = [m for m in dep.modules() if isinstance(m, B200Block)]
    assert len(blocks) == len(model.blocks) and all(b._compiled is not None for b in blocks)
    with pytest.raises(AssertionError):
        blocks[0].convert(tuple(x.shape))                    # a block converts once (convolutions.py:120-122)
    out = dep(x).float().cpu()
    ref = g["output"]
    scale = float(ref.abs().max())
    assert float((out - ref).abs().max()) <= 2e-3 * scale      # block boundaries round-trip through NCDHW fp32
    assert float((out - whole).abs().max()) <= 2e-3 * scale
    # a different batch size at run time gets its own plan instead of a silent broadcast
    x3 = torch.cat([x, x, x], 0)
    out3 = dep(x3).float().cpu()
    assert out3.shape == (3, 400) and torch.allclose(out3[2:3], out, rtol=2e-3, atol=2e-3 * scale)
    # in-place transmute of a fresh tree keeps the parameters (same state_dict values under "block." prefixes)
    m2 = TS.build_case("c1_x3d_xs", PH, g["weight_seed"], g["input_seed"])[0].cuda()
    sd = {k: v.clone() for k, v in m2.state_dict().items()}
    transmute_model(m2, "b200")
    sd2 = m2.state_dict()
    assert len(sd2) == len(sd)
    for k2, v2 in sd2.items():
        k = k2.replace(".block.", ".", 1)                    # blocks.0.block.conv.conv_t.weight -> blocks.0.conv.conv_t.weight
        assert k in sd and torch.equal(sd[k], v2), k2
    model.cpu()


def test_compiled_model_rejects_other_shapes():
    from pytorchvideo_b200.engine import compile_model
    model = TS.randomize_model(PH.x3d_xs(), seed=3).eval()
    x = torch.rand(2, 3, 4, 160, 160).cuda()
    cm = compile_model(model, x)
    cm(x)
    with pytest.raises(RuntimeError):
        cm(x[:1])                                            # would broadcast into the static buffer
    with pytest.raises(RuntimeError):
        cm([x])
