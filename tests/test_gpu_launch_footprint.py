"""Every launch of every plan touches only what it declares, and the lanes' legal orders all compute the same bits.

The float64 audits compare each op's declared output with float64 computed from its declared inputs; the multi-lane
schedule (Plan._schedule, checked by tests/test_plan_schedule.py) is built from the same declarations.  Neither sees a
kernel that writes outside its output slice (the neighbouring channels of a concat buffer another lane writes at the
same time) or reads a buffer its op does not list.  This file checks each launch against its declaration
(testing.footprint_walk): the plan's buffers are laid out twice, with guard bytes between them, as the true state
and as a canary copy.  In program order each op runs on the true state, and on the canary copy, where every element
(and guard byte) it does not declare as read holds a canary, once per canary (all-ones bytes, NaN in f16 and fp32;
0x7B bytes, large finite values).  Its declared output must come out bit-equal to the true run, and every other byte
must be untouched.  Masks and other non-float buffers,
which kernels read as counts, are never overwritten, only checked for writes.  The constants and the staged inputs
must be bit-unchanged at the end.  Each multi-lane plan also runs on one stream in two legal orders of its
happens-before graph (its highest lane as early as its waits allow, and as late), and every buffer must equal the
program-order run bit for bit.

Scope (testing.footprint_cases): every audit_catalogue case in f16 and in f32 parity mode, and the multi-lane cases
(SlowFast, Audiovisual SlowFast, the masked multipath models) also at batch 3.  This file runs the f16 rows and the
self-tests; test_gpu_launch_footprint_f32.py the f32 rows.

Self-tests, by editing the declarations of a compiled x3d_xs plan (the kernels are untouched): a convolution's
residual removed from its reads, one output TRef narrowed by 8 channels, and an SE-sum accumulator declared as written
only are each rejected, and no other op is.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit): this file 112 s, the f32 file 188 s.
  f16, 105 plans, 6715 ops checked, none skipped: 4306 implicit-GEMM / stem convolutions, 69 grouped, 17 direct,
    9 stem stream, 84 fused blocks, 392 depthwise, 154 MViT pooling convs, 215 pools, 18 temporal tap sums, 198 SE
    scale / activation, 197 SE gates and 197 SE-sum clears, 160 add + LayerNorm, 28 LayerNorm, 98 LayerNorm sets,
    60 class-token copies, 138 attention, 19 masked attention, 15 attention weights, 4 RoIAlign, 14 LSTM, the masked
    pools, defaults, reduce fusions and mask copies, and every layout conversion and copy.
  f32, 105 plans, 6889 ops checked, none skipped: 4677 direct convolutions, 392 depthwise, 154 MViT pooling convs,
    188 LayerNorm, and the same other families.
  Both legal orders of each of the 28 multi-lane plans per precision equal to program order in every buffer.
The walk found no kernel reading or writing outside its declaration.  What it and the schedule check found were
declarations: twelve kinds of op (the SE sum, gate and scale, the activation, the MViT pooling conv, max / average
pool, class-token copy and pooled LayerNorm, add + LayerNorm and attention) declared no I/O and acted as barriers, and
the depthwise convolution that accumulates the SE sums declared them as written only, while it adds onto them.  Each
now declares what its record reads and writes, and Plan._schedule orders write-after-read and write-after-write pairs
across lanes, which no current plan needs: every multi-lane plan keeps the waits it had.
"""
import collections
import os
import sys
import time

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.engine.plan import TRef  # noqa: E402

CASES = [r for r in TS.footprint_cases(bench.WORKLOADS) if TS.footprint_part(r) == "f16"]


def _flat(x):
    return list(x) if isinstance(x, (list, tuple)) else [x]


def compile_case(prec, family, case, batch):
    from pytorchvideo_b200.engine import compile_model
    if batch is None:
        m, x, extra, _ = TS.build_audit_case(family, case)
    else:
        bc = TS.BatchCase(family, case, batch)
        m, x, extra = bc.model, bc.example(bc.batch(batch)), bc.extra
    ins = [t.cuda() for t in _flat(x)]
    cm = compile_model(m, ins if isinstance(x, (list, tuple)) else ins[0], dtype=prec, use_graph=False, extra=extra)
    for s, t in zip(cm.static_in, ins):
        s.copy_(t)
    torch.cuda.synchronize()
    return cm


def run_row(prec, family, case, batch):
    t0 = time.time()
    cm = compile_case(prec, family, case, batch)
    plan = cm.plan
    lanes = sorted(set(plan.op_lane))
    orders = 0
    with torch.no_grad():
        if len(lanes) > 1:
            ref = TS.run_in_order(plan, range(len(plan.ops)))
            legal = TS.legal_orders(plan)
            assert any(o != list(range(len(plan.ops))) for o in legal)
            for order in legal:
                got = TS.run_in_order(plan, order)
                bad = [k for k, (a, b) in enumerate(zip(ref, got)) if not torch.equal(TS._bits(a), TS._bits(b))]
                assert not bad, "a legal order leaves %d buffers unlike program order (first: buffer %d)" % (
                    len(bad), bad[0])
                orders += 1
        TS.run_in_order(plan, [])
        checked, failures, skipped = TS.footprint_walk(plan, cm.static_in)
    assert not failures, "\n".join("op %d %s: %s" % f for f in failures[:20])
    assert not skipped, skipped
    assert checked == len(plan.ops)
    kinds = collections.Counter((s["route"] if s["kind"] == "conv" else s["kind"]) if s is not None else "se_zero"
                                for s in plan.op_spec)
    print("RESULT %s %s %s b%s: %d ops checked, 0 skipped, %d lanes, %d legal orders equal, %.1f s; %s" % (
        prec, family, case, batch, checked, len(lanes), orders, time.time() - t0,
        ", ".join("%s %d" % kv for kv in sorted(kinds.items()))))
    del cm, plan
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("prec,family,case,batch", CASES, ids=["%s-%s-%s-b%s" % r for r in CASES])
def test_launch_footprint(prec, family, case, batch):
    run_row(prec, family, case, batch)


@pytest.mark.gpu
def test_walk_rejects_undeclared_reads_and_writes():
    cm = compile_case("f16", "model", "x3d_xs", None)
    plan = cm.plan
    convs = [i for i, s in enumerate(plan.op_spec) if s is not None and s["kind"] == "conv"]
    res = next(i for i in convs if plan.op_spec[i]["residual"] is not None)
    se = next(i for i in convs if plan.op_spec[i]["se_sums"] is not None)
    narrow = next(i for i in convs if i not in (res, se) and plan.op_spec[i]["y"].Cp >= 16
                  and plan.op_spec[i]["residual"] is None and plan.op_spec[i]["se_sums"] is None)
    reads, writes = plan.op_io[res]
    reads.remove(plan.op_spec[res]["residual"])
    plan.op_io[se][0].remove(plan.op_spec[se]["se_sums"])
    y = plan.op_spec[narrow]["y"]
    plan.op_io[narrow][1][plan.op_io[narrow][1].index(y)] = TRef(y.buf, y.N, y.T, y.H, y.W, y.Cp - 8, Cp=y.Cp - 8,
                                                                 ch_off=y.ch_off, row_stride=y.row_stride)
    check = {res, se, narrow, res + 1, se + 1}                 # the ops after the edited ones keep passing
    with torch.no_grad():
        TS.run_in_order(plan, [])
        checked, failures, _ = TS.footprint_walk(plan, cm.static_in, check=check)
    assert checked == len(check)
    got = {i: m for i, _, m in failures}
    assert sorted(got) == sorted({res, se, narrow}), failures
    assert "declared output differ" in got[res] and "outside" not in got[res]
    assert "declared output differ" in got[se] and "outside" not in got[se]
    assert "outside its declared output changed" in got[narrow]
    for i in (res, se, narrow):
        print("RESULT self-test: %s rejected: %s" % (plan.ops[i][0], got[i][:200]))
