"""CPU: the multi-lane schedule orders every pair of launches whose declared footprints conflict.

Plan._schedule turns the ops' declared I/O (Plan.op_io) into cross-stream waits.  This file checks the result at
element level: for every plan of the audit catalogue, in f16 and f32, and for the multi-lane cases at every batch of
the batch audit's sweep, every pair of ops on different lanes whose declared footprints (testing.footprint: a TRef's
rows and channel slice, a Buf's whole buffer) share an element, at least one of them writing it (read-after-write,
write-after-read, write-after-write), must be ordered by a path of the happens-before graph (stream order within a
lane and the waits).  Two lanes writing disjoint channel slices of one concat buffer need no order; overlapping ones
do.  No op may declare no I/O.  Mutations of a SlowFast plan (a dropped wait, a concat part widened into its
neighbour, an added write-after-read across lanes) must each be rejected, naming the pair of ops.

tests/test_gpu_launch_footprint.py checks on the GPU that each launch touches only what it declares.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pytorchvideo_b200 import _lib as L  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402
from pytorchvideo_b200.engine.lower import lower_only  # noqa: E402
from pytorchvideo_b200.engine.plan import Buf, MaskRef, RawIn, TRef  # noqa: E402

# ops that may declare no I/O (each would be a full barrier across lanes): none
UNKNOWN_IO = ()

CASES = TS.footprint_cases(bench.WORKLOADS, sweep=True)
IDS = ["%s-%s-%s-b%s" % c for c in CASES]


def _plan(prec, family, case, batch):
    if batch is None:
        m, x, extra, _ = TS.build_audit_case(family, case)
    else:
        bc = TS.BatchCase(family, case, batch)
        m, x, extra = bc.model, bc.example(bc.batch(batch)), bc.extra
    plan, _ = lower_only(m, x, dtype=prec, extra=extra)
    plan._schedule()
    return plan


def _names(plan, conflicts):
    return {(plan.ops[i][0], plan.ops[j][0]) for i, j, _, _ in conflicts}


@pytest.mark.parametrize("prec,family,case,batch", CASES, ids=IDS)
def test_schedule_orders_every_conflicting_pair(prec, family, case, batch):
    plan = _plan(prec, family, case, batch)
    unknown = sorted({n for (n, _), io in zip(plan.ops, plan.op_io) if io is None})
    assert tuple(unknown) == UNKNOWN_IO, unknown
    assert (len(plan.sched["lanes"]) > 1) == TS.multi_lane_case(family, case), plan.sched["lanes"]
    bad = TS.schedule_conflicts(plan)
    assert not bad, "\n".join(m for _, _, _, m in bad[:10])
    # every buffer a record reads as a mask is one the footprint walk never fills with a canary, and every RoI box
    # tensor is a staged input, not a plan buffer
    addr = TS.address_buffers(plan)
    plan_bufs = {id(b) for b in plan.bufs}
    for (n, _), spec in zip(plan.ops, plan.op_spec):
        for key, v in (spec or {}).items():
            if isinstance(v, MaskRef) and v.buf is not None:
                assert id(v.buf) in addr, (n, key)
            if key == "rois":
                assert isinstance(v, RawIn) and id(v.tensor) not in plan_bufs, n
    for b in plan.bufs:
        if b.dt == L.PV_U8:
            assert id(b) in addr


# =====================================================================================================================
# the check rejects what it claims to reject
# =====================================================================================================================
@pytest.fixture(scope="module")
def slowfast():
    return lambda: _plan("f16", "model", "slowfast_r50", None)


def _index(plan, name):
    return [n for n, _ in plan.ops].index(name)


def test_a_dropped_wait_is_named(slowfast):
    plan = slowfast()
    assert not TS.schedule_conflicts(plan)
    w = _index(plan, "blocks.1.multipathway_fusion.conv_fast_to_slow")
    r = _index(plan, "blocks.2.multipathway_blocks.0.res_blocks.0.branch1")
    assert w in plan.sched["waits"][r]
    waits = [list(x) for x in plan.sched["waits"]]
    waits[r].remove(w)
    bad = TS.schedule_conflicts(plan, waits)
    assert (w, r, "RAW") in {b[:3] for b in bad}, bad
    msg = next(m for i, j, _, m in bad if (i, j) == (w, r))
    assert plan.ops[w][0] in msg and plan.ops[r][0] in msg


def test_a_widened_concat_part_is_named_and_then_ordered(slowfast):
    plan = slowfast()
    fuse = _index(plan, "blocks.1.multipathway_fusion.conv_fast_to_slow")
    cat = plan.op_spec[fuse]["y"].buf
    # the Slow pathway's writer of the same concat buffer: its channels [0, 256) meet the lateral's [256, 288) once
    # widened by 8 channels
    slow = next(i for i, io in enumerate(plan.op_io) if plan.op_lane[i] == 0 and io is not None
                and any(isinstance(t, TRef) and t.buf is cat for t in io[1]))
    y = plan.op_spec[slow]["y"]
    assert y.ch_off == 0 and y.Cp == plan.op_spec[fuse]["y"].ch_off
    y.Cp += 8
    bad = TS.schedule_conflicts(plan)
    assert [(b[0], b[1], b[2]) for b in bad] == [(slow, fuse, "WAW")], bad
    assert plan.ops[slow][0] in bad[0][3] and plan.ops[fuse][0] in bad[0][3]
    # with the real footprints Plan._schedule orders the overlapping writers
    plan._schedule()
    assert slow in plan.sched["waits"][fuse] and not TS.schedule_conflicts(plan)
    y.Cp -= 8
    plan._schedule()
    assert slow not in plan.sched["waits"][fuse]       # disjoint slices stay concurrent


def test_an_added_write_after_read_is_named_and_then_ordered(slowfast):
    plan = slowfast()
    hb = TS.happens_before(plan)
    # a Slow-lane read of a Fast-produced tensor: the lateral conv's input is read on lane 1; pick a lane-0 reader of
    # the stage's concat buffer and a later lane-1 op that nothing orders after it
    r = _index(plan, "blocks.2.multipathway_blocks.0.res_blocks.0.branch1")
    x = plan.op_spec[r]["x"]
    w = next(j for j in range(r + 1, len(plan.ops)) if plan.op_lane[j] == 1 and hb[j].get(0, -1) < r)
    plan.op_io[w][1].append(x)
    bad = TS.schedule_conflicts(plan)
    assert (r, w, "WAR") in {b[:3] for b in bad}, bad
    msg = next(m for i, j, h, m in bad if (i, j, h) == (r, w, "WAR"))
    assert plan.ops[r][0] in msg and plan.ops[w][0] in msg
    plan._schedule()
    assert not TS.schedule_conflicts(plan)
    assert any(j >= r and plan.op_lane[j] == 0 for j in plan.sched["waits"][w])


def test_an_in_place_op_across_lanes_waits_for_the_other_lanes_reader():
    """Plan._schedule on a hand-built plan: lane 0 writes x, lane 1 reads it, then lane 0 updates x in place.  The
    in-place op must wait for lane 1's read (write-after-read), which read-after-write alone does not give."""
    from pytorchvideo_b200.engine.plan import Plan
    plan = Plan("cpu")
    x = plan.new_tensor(1, 1, 1, 4, 8)
    y = plan.new_tensor(1, 1, 1, 4, 8)
    noop = lambda s: None                                    # noqa: E731
    plan.add("produce", noop, reads=(), writes=(x,))
    plan.lane = 1
    plan.add("read", noop, reads=(x,), writes=(y,))
    plan.lane = 0
    plan.add("in_place", noop, reads=(x,), writes=(x,))
    plan._schedule()
    assert plan.sched["waits"] == [[], [0], [1]]
    assert not TS.schedule_conflicts(plan)
    assert [b[:3] for b in TS.schedule_conflicts(plan, [[], [0], []])] == [(1, 2, "WAR")]


def test_footprints_of_concat_slices_token_rows_and_buffers():
    b = Buf(2 * 3 * 24, L.PV_F16)
    a = TRef(b, 2, 1, 1, 3, 16, Cp=16, ch_off=0, row_stride=24)
    c = TRef(b, 2, 1, 1, 3, 8, Cp=8, ch_off=16, row_stride=24)
    ma, mc = TS.footprint(a).mask(b), TS.footprint(c).mask(b)
    assert int(ma.sum()) == 6 * 16 and int(mc.sum()) == 6 * 8 and not bool((ma & mc).any())
    assert bool((ma | mc).all())
    wide = TRef(b, 2, 1, 1, 3, 24, Cp=24, ch_off=0, row_stride=24)
    assert bool((TS.footprint(wide).mask(b) & mc).any())
    # token rows 1.. of each sample (a pooled token tensor behind its class row)
    rows = TS.footprint(c, slice(1, None)).mask(b).view(2, 3, 24)
    assert not bool(rows[:, 0].any()) and bool(rows[:, 1:, 16:].all()) and not bool(rows[:, 1:, :16].any())
    assert bool(TS.footprint(b).mask(b).all())
    # W-padded stem rows: the physical rows
    p = Buf(1 * 2 * 3 * 12 * 4 + 64 * 4, L.PV_F16)
    s = TRef(p, 1, 2, 3, 5, 3, Cp=4)
    s.padw = (4, 12)
    m = TS.footprint(s).mask(p)
    assert int(m.sum()) == 2 * 3 * 12 * 4 and bool(m[:2 * 3 * 12 * 4].all())


def test_footprint_cases_cover_the_catalogue_and_the_multi_lane_sweep():
    cat = TS.audit_catalogue(bench.WORKLOADS)
    gpu = TS.footprint_cases(bench.WORKLOADS)
    assert {(p, f, c) for p, f, c, b in gpu if b is None} == {(p, f, c) for p in ("f16", "f32") for f, c, _ in cat}
    multi = {(f, c) for f, c, _ in cat if TS.multi_lane_case(f, c)}
    assert multi and {(p, f, c) for p, f, c, b in gpu if b == 3} == {(p, f, c) for p in ("f16", "f32") for f, c in multi}
    # every case of the GPU walk runs in exactly one of its files
    parts = [TS.footprint_part(r) for r in gpu]
    assert set(parts) == set(TS.FOOTPRINT_PARTS)
    assert len(gpu) == len(set(gpu))
