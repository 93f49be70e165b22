"""Every launch of the seven bench.py workloads against float64, at the shapes the benchmark runs.

The kernel matrices test each compiled instance on small synthetic shapes.  This file checks the launches the
benchmark actually makes: concat buffers written through retargeted TRefs, Block-N choices at real M, long persistent
tile walks, the window-mode and stem-stream inputs at 224^2, SE sums at batch 32 and the fp32 MViT trunk.  Each op
of a plan carries a record of what it computes (``Plan.op_spec``); the audit walks the plan on one stream, reads each
op's inputs just before it runs (so in-place ops are checked against their own operands, and errors do not compound
from op to op), runs it, asserts that the launched instances belong to the family the record implies, and compares
the output with the same operation in float64 on the GPU under the bounds of the kernel matrices (conv, fused block
and attention bounds of testing.py, the CUDA-core bounds of test_gpu_simt_matrix.py; bit-exact for layout
conversions, max pooling, copies and add_pos_cls).  Pad channels of every output must be zero, and channels of a
shared concat buffer outside the op's slice must be left as they were.

The kernels run the full batch.  The reference and the comparison cover clips 0, B // 2 and B - 1: eval forward has
no coupling between clips, and the three clips cover the first tiles, the last (ragged) tiles and the middle of
every launch's tile walk while keeping the float64 copies (moved to the host for the comparison) to a few minutes
for the file.

After the audit, the same plan is captured as the benchmark runs it (several lanes on side streams, PDL, one CUDA
graph) and replayed; every plan buffer must equal the single-stream run bit for bit, also after a replay on other
inputs (a lane reading a buffer before its producer finished would see the other input's values).

CPU tests: every launch of every workload has a record the audit checks, the read / write declarations that order
the lanes cover every buffer a record reads and writes, and sampled records agree with their torch modules.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit): 748 of the 778 launches audited (the other 30 are the
SE-sum clears of the two X3D plans, which compute no value).  Largest err / tol per family over the seven workloads:
conv igemm / gather / stem 0.996, depthwise 0.996, fused block 0.581, stem stream 0.857, temporal tap sum 0.989, average pool 0.980, scale_act
0.999, se_gate 0.005, head 0.010, LayerNorm 0.985 / 0.986 (sets), add_layernorm 0.986, attention 0.211, MViT
pooling conv 0.996; layout conversions, max pooling, copies, add_pos_cls and the add_layernorm sums bit-exact.  Graph
replay equal to the single-stream run in every buffer of every workload.  The file took 5.5 minutes (csn_r101 86 s,
mvit_base_16x4 71 s, r2plus1d_r50 53 s, slowfast_r50 43 s, x3d_m 29 s, slow_r50 26 s, x3d_xs 3 s, plus set-up).
"""
import os
import sys
import time

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pytorchvideo_b200 import _lib as L  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.engine.plan import Buf, TRef  # noqa: E402

WORKLOADS = sorted(bench.WORKLOADS)


def build_workload(name, use_graph=False, batch=None):
    from pytorchvideo_b200.engine import compile_model
    model, B, T, H, W, is_sf = bench.build_model_and_inputs(name, batch)

    def inputs(seed):
        x = bench.make_inputs(B, T, H, W, is_sf, seed=seed)
        return [t.cuda() for t in (x if is_sf else [x])]
    ins, alt = inputs(42), inputs(43)           # bench.py's inputs, and a second set for the replay
    cm = compile_model(model, ins if is_sf else ins[0], dtype="f16", use_graph=use_graph)
    return cm, ins, alt, B


def stage(cm, ins):
    for s, t in zip(cm.static_in, ins):
        s.copy_(t)


# =====================================================================================================================
# GPU: the audit and the graph replay, per workload
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("name", WORKLOADS)
def test_workload_audit_and_graph_replay(name):
    t0 = time.time()
    cm, ins, alt, B = build_workload(name)
    plan = cm.plan
    stage(cm, ins)
    torch.cuda.synchronize()
    with torch.no_grad():
        failures, stats = TS.audit_plan(plan, TS.audit_clips(B))
    t_audit = time.time() - t0
    n_checked = sum(v[0] for v in stats.values())
    insts = set().union(*(v[2] for v in stats.values())) if stats else set()
    print("RESULT %s: %d launches, %d audited, %d instances, %.0f s; largest err/tol per family: %s" % (
        name, len(plan.ops), n_checked, len(insts), t_audit,
        ", ".join("%s %d x %.3f" % (k, v[0], v[1]) for k, v in sorted(stats.items()))))
    assert not failures, "\n".join("op %d %s: %s" % f for f in failures[:20])
    assert n_checked + sum(1 for s in plan.op_spec if s is None) == len(plan.ops)

    # ---- graph replay against the single-stream run, buffer for buffer
    lanes, nbufs = TS.check_graph_replay(cm, ins, alt)
    print("RESULT %s: graph replay (%d lanes) equals the single-stream run in all %d buffers, %.0f s in all" % (
        name, lanes, nbufs, time.time() - t0))
    del cm, plan
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_audit_rejects_a_corrupted_tile_and_its_references_agree_with_the_cpu():
    """Self-checks on x3d_xs: one 128-row tile of one convolution output moved by 8 f16 ulp after its launch fails
    the audit under that op's name; and the float64 reference of the first op of each kind agrees between the GPU
    and the CPU to 1e-12 relative, whatever algorithm cuDNN picks on the GPU."""
    cm, ins, _, B = build_workload("x3d_xs")
    plan = cm.plan
    target = next(i for i, s in enumerate(plan.op_spec) if s is not None and s["kind"] == "conv"
                  and s["route"] == "tcgen05" and s["y"].N * s["y"].npos >= 4 * 128 and i > 2)

    def corrupt(i, spec):
        if i == target:
            y = spec["y"]
            rows = TS.full_rows(y).reshape(-1, y.row_stride)
            tile = rows[128:256, y.ch_off:y.ch_off + y.C]
            tile.view(torch.int16).add_(8)
    stage(cm, ins)
    cpu_check = {}
    with torch.no_grad():
        failures, _ = TS.audit_plan(plan, [0], corrupt=corrupt, cpu_check=cpu_check)
    names = [f[1] for f in failures]
    assert names == [plan.ops[target][0]], failures
    print("RESULT self-check: corrupted %s rejected (%s); GPU vs CPU float64 references: %s" % (
        names[0], failures[0][2][:120], cpu_check))
    assert cpu_check and all(r <= 1e-12 for r in cpu_check.values()), cpu_check


# =====================================================================================================================
# CPU: records, declared I/O, module agreement
# =====================================================================================================================
_PLANS = {}


def _lowered(name):
    if name not in _PLANS:
        from pytorchvideo_b200.engine.lower import lower_only
        model, B, T, H, W, is_sf = bench.build_model_and_inputs(name)
        shape = (B, 3, T, H, W)
        x = torch.empty(shape)
        plan, _ = lower_only(model, TS.slowfast_inputs(x) if is_sf else x)
        _PLANS.clear()
        _PLANS[name] = (plan, model)
    return _PLANS[name]


EXPECTED_LAUNCHES = {"slowfast_r50": 103, "x3d_m": 135, "x3d_xs": 135, "slow_r50": 58, "csn_r101": 109,
                     "r2plus1d_r50": 73, "mvit_base_16x4": 165}


@pytest.mark.parametrize("name", WORKLOADS)
def test_every_launch_has_a_checked_record(name):
    plan, _ = _lowered(name)
    assert len(plan.op_spec) == len(plan.ops) == EXPECTED_LAUNCHES[name]
    missing = [n for (n, _), s in zip(plan.ops, plan.op_spec)
               if not TS.supported(s) and not n.endswith(TS.NO_VALUE_SUFFIXES)]
    assert not missing, missing
    for (n, _), s in zip(plan.ops, plan.op_spec):
        if s is None:
            continue
        for t in TS.record_io(s)[0] + TS.record_io(s)[1]:
            assert isinstance(t, (TRef, Buf)), (n, t)


@pytest.mark.parametrize("name", WORKLOADS)
def test_declared_io_covers_the_records(name):
    plan, _ = _lowered(name)
    assert not TS.io_problems(plan)


@pytest.mark.parametrize("case", sorted(c for c, v in TS.AUDIO_CASES.items() if v[2][0] == "avsf"))
def test_declared_io_covers_the_records_audio(case):
    """AVSlowFast lanes read across pathways: a missing declaration would be a cross-lane race."""
    from pytorchvideo_b200.engine.lower import lower_only
    from pytorchvideo_b200 import models as M
    m, x = TS.build_audio_case(case, M, seed=2024)
    plan, _ = lower_only(m, x)
    assert len(set(plan.op_lane)) > 1
    assert not TS.io_problems(plan)


_ACT_OF = {"ReLU": L.ACT_RELU, "SiLU": L.ACT_SWISH, "Swish": L.ACT_SWISH, "GELU": L.ACT_GELU}


@pytest.mark.parametrize("name", WORKLOADS)
def test_records_agree_with_their_modules(name):
    plan, model = _lowered(name)
    mods = dict(model.named_modules())
    checked = 0
    for (n, _), s in zip(plan.ops, plan.op_spec):
        m = mods.get(n)
        if s is None or s["kind"] != "conv" or type(m).__name__ != "Conv3d":
            continue
        assert s["stride"] == tuple(m.stride) and s["padding"] == tuple(m.padding), n
        assert s["dilation"] == tuple(m.dilation), n
        # grouped convolutions the library does not take run as dense block-diagonal convolutions
        assert s["groups"] == m.groups or (s["groups"] == 1 and s["weight"].shape[1] == m.in_channels), n
        assert tuple(s["weight"].shape[0:1]) == (m.out_channels,) and s["x"].C == m.in_channels, n
        parent, _, leaf = n.rpartition(".")
        # conv_a's activation is fused into it in every family (conv_b's may follow an SE block instead)
        act = getattr(mods.get(parent), "act_a", None) if leaf == "conv_a" else None
        if act is not None and type(act).__name__ in _ACT_OF:
            assert s["act"] == _ACT_OF[type(act).__name__], n
        checked += 1
    for (n, _), s in zip(plan.ops, plan.op_spec):
        m = mods.get(n)
        if s is not None and s["kind"] == "conv" and type(m).__name__ == "Linear":
            assert tuple(s["weight"].shape) == (m.out_features, m.in_features, 1, 1, 1), n
            assert (s["stride"], s["padding"], s["groups"]) == ((1, 1, 1), (0, 0, 0), 1), n
            checked += 1
        if s is not None and s["kind"] in ("token_conv", "pool") and s.get("modules"):
            t3 = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v,) * 3       # noqa: E731
            for m in s["modules"]:                      # pool_k and pool_v of a fused K | V pool
                assert t3(m.stride) == tuple(s["stride"]) and t3(m.padding) == tuple(s["padding"]), n
                assert t3(m.kernel_size) == tuple(s["weight"].shape[2:] if s["kind"] == "token_conv" else s["kernel"]), n
            checked += 1
        if s is not None and s["kind"] == "fused_block":
            for mod, w in zip(s["modules"], (s["wa"], s["wb"], s["wc"], s["ws"])):
                assert (mod is None and w is None) or mod.weight is w, n
            ca, cb = s["modules"][:2]
            assert s["kt"] == ca.kernel_size[0] and s["sb"] == cb.stride[1], n
            checked += 1
    assert checked >= 10, checked
