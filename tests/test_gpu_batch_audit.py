"""Every model plan at other batch sizes: each launch against float64 on every clip, and each clip's bits invariant
under reordering the batch and against the batch-1 plan.

The batch size decides how the kernels split their work: the tensor-core conv tile box and BLOCK_N (pv_igemm.cu,
pv_igemm_gather.cu), the persistent grid and the epilogue buffer parity each CTA ends on, the fused Fast-pathway block
tiling (fb_plan in pv_fastblock.cu), the SlowFast Fast-stem route (plan.py: the temporal-streaming kernel once
N * Ho * cdiv(Wo, 128) reaches the SM count, between batch 1 and 2 at 224^2), and the CUDA-core kernels' row tiles.
test_gpu_model_audit.py and test_gpu_workload_audit.py audit each plan at one batch and on three clips.  This file runs
the sweep of testing.batch_sweep, one test per (precision, case, batch):
  - the seven bench.py architectures in f16 at batch 2 and 3 (x3d_xs: 1 and 3) with checks (a), (b), (c), and at the
    bench batch with (b) and (c) (the workload audit runs (a) there);
  - every other f16 case of the model audit's catalogue at batch 3, with (a), (b), (c);
  - x3d_xs, mvit_base_8x112, the masked and the detection cases in f32 parity mode at batch 3, with (a), (b), (c);
  - the self-supervised trunks (the SimCLR video case's Slow-R50 + 2048-2048-128 BatchNorm1d projector as one
    EmbeddingChain plan with fused rows, and the chain MoCo v2's slow_r50 case compiles for its key encoder) in f16
    and f32 at batch 1, 2 and 3, with (a), (b), (c).
Inputs come from testing.BatchCase: clip j is the same tensor at every batch (a pool drawn once, sliced), the clips
differ from one another, masks are per-clip rows, and detection boxes carry their clip's index (clip 1 has none).

  (a) float64: testing.audit_plan on every clip of the batch.
  (b) position invariance: the plan runs op by op on X and on X with its clips rotated by one (masks and box indices
      with them); for every op with a record, clip c's rows of every operand it writes must be bit-equal at its new
      position, wherever the op read bit-equal rows (the first op that breaks invariance is the one named).  With
      no failure every op must have read bit-equal rows on every clip: an op that did not is a failure too.
  (c) batch-size invariance: the same against the batch-1 plan of each clip, ops matched by name: where an op
      launched the same instance names at both batches and read bit-equal rows for clip c, it must write bit-equal
      rows for clip c.  Instance names carry BLOCK_N and the k-block width, so an op whose BLOCK_N changes with the
      batch makes no claim (check (a) covers it at both batches); a change of tile box, m_tiles or grid does not
      exempt it.  Every other op must either be held or read a buffer that the data flow of an exempt op wrote.
The rows compared are the rows each op reads and writes, in the value channels of each operand.  They come from
testing.record_rows and token_span, the slicing the float64 audit uses: a pooled token tensor without its class row,
which another op writes, and a layernorm_sets without its output's class row, which it takes from x.  They are hashed
on the GPU (testing.row_digests).  An operand is per RoI by the plan's data flow from a RoIAlign's boxes, not by its
row count.  BATCH_DEPENDENT lists kernels whose bits may depend on the batch by design.

CPU tests: the sweep crosses the Fast-stem route (threshold from plan.H100_SXM_SMS), the fused Fast-block tiling of
each swept batch is pinned, and (test_gpu_model_audit.py) every swept (case, batch) lowers to records the audit checks.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit).  The 146 sweep rows take 49 minutes of test time in all
(the sum of the times the rows print), so testing.batch_sweep_part splits them over five files.  By the per-row times
they take about 9 min (this file: the bench architectures but csn_r101, and the self-check), 11 min
(test_gpu_batch_audit_models.py: csn_r101 and the other f16 model cases), 11 min (_families: grouped, hub-tail,
detection and Non-local in f16), 8 min (_layers: audio, efficient, MViT variants and masked in f16, and the f32 rows)
and 8 min (_ssl: the trunks in both precisions).  Longest rows:
slowfast_16x8_r101_50_50 b3 256 s, csn_r101_w8 b3 238 s, csn_r101 b3 195 s, mvit_base_16x4 b3 145 s,
mvit_base_32x3 b3 130 s, csn_r101 b2 126 s.
  (a) float64 on every clip: 6317 f16 and 1070 f32 launches audited (the sum of each plan's launches, not launches
      times clips).  Largest err / tol per family at the new batches:
    f16: conv igemm / gather / stem 0.997, grouped 0.995, direct 0.990, depthwise 0.997, fused block 0.840, stem
      stream 0.884, temporal tap sum 0.994, average pool 0.991, scale_act 0.999, se_gate 0.006, head 0.014, LayerNorm
      0.985 / 0.987 (sets), add_layernorm 0.986, MViT pooling conv 0.996, channel affine 0.997, attention 0.467,
      masked attention 0.262, attention weights 0.037, RoIAlign 0.998, masked average / sum 0.990, reduce fusion
      0.979, LSTM 0.872.
    f32: direct 0.209, depthwise 0.201, average pool 0.065, scale_act 0.672, se_gate 0.005, LayerNorm 0.037 / 0.041
      (sets), MViT pooling conv 0.274, attention 0.015, masked attention 0.021, attention weights 0.039, RoIAlign
      0.281, masked average / sum 0.033, reduce fusion 0.015, LSTM 0.092.
    Layout conversions, copies, token input, masked max pooling, learned defaults, max pooling and add_pos_cls are
    bit-exact.
  (b), (c) per case and batch: ops held bitwise by (b) / ops with a record, then ops held by (c), then ops exempt
  from (c).  An op counts as held when it read bit-equal rows on every clip; in (c) the rest read what an exempt
  op's data flow wrote.  Rows marked * were measured with the checks as they stand: every op held in (b), and no op in
  (c) neither held, exempt nor downstream of an exempt op.  The unmarked rows were measured with an earlier form of
  the checks.  That form digested whole token tensors and did not assert that every op was held.  In it, the token
  models held fewer ops in (b), e.g. mvit_base_16x4 147 of 165.  Each missing op was a layernorm_sets (or an op
  after one) that seemed to read its output's class row, stale from the previous run.  The kernel does not read that
  row.  The other unmarked rows have no class token, so their counts do not depend on the change.
    f16: acoustic_r50 b3 57/57 45 12; acoustic_r50_k3 b3 57/57 57 0; avg b3 56/56 56 0*;
      avsf_r18_norm_none b3 78/78 74 4; avsf_r18_sigmoid b3 78/78 74 4; avsf_r50 b3 170/170 66 42*;
      avsf_r50_b8_f16grid b3 170/170 66 42; block_bias_no_bn b3 7/7 7 0; block_hswish b3 6/6 6 0;
      block_hswish_se b3 8/8 8 0; block_no_residual b3 7/7 7 0; bn_block b3 14/14 14 0*; bn_mvit_b b3 111/111 96 15*;
      bn_mvit_b_fused b3 111/111 96 15*; bn_small b3 43/43 43 0*; c2d_r50 b3 59/59 39 20; chain b3 11/11 11 0;
      conv_3x1x1_hswish b3 3/3 3 0; conv_5x1x1_dw_hswish b3 3/3 3 0; conv_dw_swish b3 3/3 3 0;
      conv_pw_hswish b3 3/3 3 0; conv_t1_relu b3 3/3 3 0;
      csn_r101 b2 109/109 108 1, b3 109/109 82 27, b8 109/109 82 27; csn_r101_w8 b3 109/109 82 27;
      default b3 3/3 3 0; dot_product_nopool_64_256 b3 5/5 5 0; dot_product_pool_32_64 b3 7/7 7 0;
      embedding_chain b1 59/59 59 0, b2 59/59 47 12, b3 59/59 36 23; encoder_1 b3 11/11 11 0;
      encoder_2 b3 18/18 18 0; encoder_nomask b3 10/10 10 0; head_none b3 51/51 51 0*; i3d_nln b3 84/84 54 30*;
      i3d_r50 b3 59/59 39 20; lstm_bi b3 4/4 4 0; lstm_bi_t1 b3 4/4 4 0; lstm_nomask b3 4/4 4 0; lstm_uni b3 4/4 4 0;
      m_b1 b3 120/120 87 33; mha b3 7/7 7 0; mha_d128 b3 7/7 7 0; mha_d32_t1 b3 7/7 7 0; mha_nomask b3 6/6 6 0;
      moco_key b1 60/60 60 0, b2 60/60 48 12, b3 60/60 37 23; multipath_concat b3 14/14 14 0;
      multipath_max b3 15/15 15 0; multipath_prod b3 15/15 15 0; multipath_sum b3 15/15 15 0;
      multipath_temporal_concat b3 14/14 14 0; mvit_base_16 b3 165/165 157 8*;
      mvit_base_16x4 b2 165/165 144 21*, b3 147/165 125 21, b8 146/165 121 25; mvit_base_32x3 b3 165/165 161 4*;
      mvit_base_8x112 b3 165/165 157 8*; pool_avg b3 3/3 3 0; pool_avg_nomask b3 3/3 3 0; pool_first_bn b3 63/63 63 0*;
      pool_first_bn_avg b3 59/59 59 0*; pool_first_ln b3 68/68 68 0*; pool_max b3 3/3 3 0; pool_max_t1 b3 3/3 3 0;
      pool_sum b3 3/3 3 0; posenc b3 3/3 3 0; r2plus1d_r50 b2 73/73 72 1, b3 73/73 51 22, b8 73/73 51 22;
      s_b1 b3 120/120 118 2; separable_cat b3 5/5 5 0; separable_sum b3 5/5 5 0;
      slow_r50 b2 58/58 46 12, b3 58/58 35 23*, b8 58/58 30 28; slow_r50_detection b3 60/60 46 14;
      slow_r50_detection_sigmoid b3 61/61 57 4; slow_r50_g32 b3 58/58 45 13;
      slowfast_16x8_r101_50_50 b3 205/205 4 56; slowfast_r101 b3 205/205 4 88;
      slowfast_r50 b2 103/103 4 21*, b3 103/103 4 37, b8 103/103 4 42; slowfast_r50_detection b3 105/105 4 23*;
      slowfast_r50_g b3 119/119 4 27; softmax_pool_1024_512 b3 7/7 7 0; softmax_pool_32_128 b3 7/7 7 0;
      softmax_pool_32_64 b3 7/7 7 0; softmax_pool_512_256 b3 7/7 7 0; softmax_pool_norm_none b3 7/7 7 0;
      softmax_pool_ragged b3 7/7 7 0; tokens b3 27/27 23 4*; tokens_no_cls b3 27/27 23 4*; x3d_l b3 235/235 186 49;
      x3d_m b2 120/120 109 11, b3 120/120 87 33*, b32 120/120 78 42*; x3d_s b3 120/120 118 2;
      x3d_xs b1 120/120 120 0, b3 120/120 120 0, b8 120/120 118 2; xs_b2 b3 120/120 120 0;
      xs_b8_f16grid b3 120/120 120 0; xs_head_hswish b3 120/120 120 0; xs_head_relu b3 120/120 120 0;
      xs_head_swish b3 120/120 120 0; xs_no_head b3 116/116 116 0
    f32: chain b3 11/11 11 0*; default b3 3/3 3 0*; embedding_chain b1 59/59 59 0, b2 59/59 59 0, b3 59/59 59 0;
      encoder_1 b3 11/11 11 0*; encoder_2 b3 18/18 18 0*; encoder_nomask b3 10/10 10 0*; lstm_bi b3 4/4 4 0*;
      lstm_bi_t1 b3 4/4 4 0*; lstm_nomask b3 4/4 4 0*; lstm_uni b3 4/4 4 0*; mha b3 7/7 7 0*; mha_d128 b3 7/7 7 0*;
      mha_d32_t1 b3 7/7 7 0*; mha_nomask b3 6/6 6 0*; moco_key b1 60/60 60 0, b2 60/60 60 0, b3 60/60 60 0;
      multipath_concat b3 14/14 14 0*; multipath_max b3 15/15 15 0*; multipath_prod b3 15/15 15 0*;
      multipath_sum b3 15/15 15 0*; multipath_temporal_concat b3 14/14 14 0*; mvit_base_8x112 b3 165/165 165 0*;
      pool_avg b3 3/3 3 0*; pool_avg_nomask b3 3/3 3 0*; pool_max b3 3/3 3 0*; pool_max_t1 b3 3/3 3 0*;
      pool_sum b3 3/3 3 0*; posenc b3 3/3 3 0*; slow_r50_detection b3 60/60 60 0*;
      slow_r50_detection_sigmoid b3 61/61 61 0*; slowfast_r50_detection b3 120/120 120 0*; x3d_xs b3 120/120 120 0*
  Exempt from (c): 1090 op launches (over all cases and batches) whose conv3d_igemm_kernel BLOCK_N differs from
  batch 1 (e.g. <128,128> at batch 3 against <64,128> at batch 1), 29 conv3d_igemm_gather_kernel BLOCK_N changes, and
  9 Fast stems that flip from conv3d_stem_rows_kernel (batch 1) to conv3d_stem_stream_kernel.  No other op changed
  instance.
  Self-check (test_invariance_checks_name_a_corrupted_tile): blocks.1.res_blocks.0.branch1 corrupted on clip 1 is
  named by (b) and by (c), and no other op is.
Findings: in every row measured, no kernel read or reduced across clips or batch slots. Each op that kept its
instances gave the same bits for a clip at every position and batch, so BATCH_DEPENDENT stays empty. One launch
failed: the image MViT (hub_tail mvit_base_16) at batch 3. pv_dwplane_fwd encoded a TMA tensor map for its stride-4
K|V pool, a path that reads x straight from global memory and never uses the map. The box was chosen without the
shared-memory budget, and the driver rejected it (CUDA_ERROR_INVALID_VALUE). The map is now encoded only for strides
1 and 2. test_gpu_hub_tail.py has the row h56_s4_c192_n3 for this shape.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pytorchvideo_b200 import testing as TS  # noqa: E402

ALL = TS.batch_sweep(bench.WORKLOADS)
POOL = TS.batch_pools(ALL)
SWEEP = [r for r in ALL if TS.batch_sweep_part(r, bench.WORKLOADS) == "workloads"]

# Kernels whose bits may depend on the batch by design (a reduction split by grid size): instance prefix -> reason
# and DESIGN.md section.  (c) makes no claim for an op that launched one; (a) still checks it.  None so far; every
# file of the batch audit passes this table.
BATCH_DEPENDENT = {}


def run_row(prec, family, case, B, checks):
    for line in TS.run_batch_audit(prec, family, case, B, checks, POOL[(family, case)], tuple(BATCH_DEPENDENT)):
        print(line)


# =====================================================================================================================
# GPU: the sweep's bench architectures (csn_r101 runs in test_gpu_batch_audit_models.py)
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("prec,family,case,B,checks", SWEEP, ids=["%s-%s-%s-b%d" % r[:4] for r in SWEEP])
def test_batch_audit(prec, family, case, B, checks):
    run_row(prec, family, case, B, checks)


@pytest.mark.gpu
def test_invariance_checks_name_a_corrupted_tile():
    """x3d_xs f16 at batch 3: the last 64-row tile of clip 1 of one convolution output scaled by 1 + 2^-10 after its
    launch.  Applied in the first of the two position runs, check (b) names that op and no other; applied in the
    batch-3 run only, check (c) names that op and no other."""
    prec, B = "f16", 3
    bc = TS.batch_case("model", "x3d_xs", POOL[("model", "x3d_xs")])
    ins = bc.batch(B)
    cm = TS.batch_compile(bc, ins, prec)
    plan = cm.plan
    rows = TS.clip_rows_fn(B)
    clean = TS.batch_digests(cm, ins, rows)
    held = set(TS.invariance_failures(clean, TS.merge_single(TS.batch_single_digests(prec, bc, B)))[1])
    seen = {}
    target = None
    for i, ((name, _), s) in enumerate(zip(plan.ops, plan.op_spec)):
        key = (name, seen.get(name, 0))
        seen[name] = key[1] + 1
        if (target is None and i > 2 and key in held and s is not None and s["kind"] == "conv"
                and s["route"] == "tcgen05" and s["y"].npos >= 2 * 64):
            target = (i, key)
    assert target is not None

    def corrupt(i, spec):
        if i == target[0]:
            y = spec["y"]
            r = TS.full_rows(y)[1].reshape(-1, y.row_stride)
            r[-64:, y.ch_off:y.ch_off + y.C] *= 1 + 2.0 ** -10
    bad = TS.batch_digests(cm, ins, rows, corrupt)
    rot = TS.batch_digests(cm, bc.batch(B, rotate=True), TS.clip_rows_fn(B, perm=[(c + 1) % B for c in range(B)]))
    fb = TS.invariance_failures(bad, rot)[0]
    assert [f[0] for f in fb] == [target[1]] and fb[0][1] == [1], fb
    fc = TS.invariance_failures(bad, TS.merge_single(TS.batch_single_digests(prec, bc, B)))[0]
    assert [f[0] for f in fc] == [target[1]] and fc[0][1] == [1], fc
    print("RESULT self-check: %s named by (b) and (c), no other op" % target[1][0])


# =====================================================================================================================
# CPU: the sweep crosses routes and tilings, and is split over the files
# =====================================================================================================================
def test_every_sweep_row_runs_in_one_file():
    parts = [TS.batch_sweep_part(r, bench.WORKLOADS) for r in ALL]
    assert set(parts) == set(TS.BATCH_AUDIT_PARTS)
    for part in TS.BATCH_AUDIT_PARTS:
        name = "test_gpu_batch_audit%s.py" % ("" if part == "workloads" else "_" + part)
        assert os.path.exists(os.path.join(ROOT, "tests", name)), name


_SF_BATCHES = sorted({1} | {r[3] for r in ALL if r[2] == "slowfast_r50"})


@pytest.fixture(scope="module")
def slowfast_plans():
    from pytorchvideo_b200.engine.lower import lower_only
    bc = TS.BatchCase("model", "slowfast_r50", max(_SF_BATCHES))
    return {B: lower_only(bc.model, bc.batch(B))[0] for B in _SF_BATCHES}


def test_sweep_crosses_the_fast_stem_route(slowfast_plans):
    """SlowFast's Fast stem takes the factored route at batch 1 and the temporal-streaming kernel from the batch where
    N * Ho * cdiv(Wo, 128) reaches plan.H100_SXM_SMS; the sweep's batches and their batch-1 plans lie on both sides."""
    from pytorchvideo_b200.engine.plan import H100_SXM_SMS
    routes = {}
    for B, plan in slowfast_plans.items():
        taps = [s for (n, _), s in zip(plan.ops, plan.op_spec) if n.endswith(".taps")]
        assert len(taps) == 1 and len([n for n, _ in plan.ops if n.endswith(".tapsum")]) == 1, B
        y = taps[0]["y"]
        stream = B * y.H * -(-y.W // 128) >= H100_SXM_SMS
        assert taps[0]["route"] == ("stem_stream" if stream else "tcgen05"), (B, taps[0]["route"])
        routes[B] = taps[0]["route"]
    assert routes[1] == "tcgen05" and all(routes[B] == "stem_stream" for B in _SF_BATCHES if B > 1), routes


# (th, tw, frames per CTA) of the seven fused Fast-pathway blocks on 132 SMs, per swept batch
FUSED_TILINGS = {
    1: [(6, 8, 4), (6, 8, 4), (6, 8, 4), (7, 8, 4), (8, 12, 4), (8, 12, 4), (8, 12, 4)],
    2: [(8, 12, 4), (8, 14, 4), (8, 14, 4), (4, 8, 4), (8, 14, 4), (8, 14, 4), (8, 14, 4)],
    3: [(8, 14, 4), (14, 14, 4), (14, 14, 4), (7, 8, 6), (10, 14, 4), (10, 14, 4), (10, 14, 4)],
    8: [(8, 14, 7), (14, 14, 7), (14, 14, 7), (4, 8, 11), (10, 14, 6), (10, 14, 6), (10, 14, 6)],
}


def _fused_tilings(plan):
    import ctypes as C
    from pytorchvideo_b200 import _lib as L
    out = []
    for s in plan.op_spec:
        if s is None or s["kind"] != "fused_block":
            continue
        x = s["x"]
        d = plan.fused_bottleneck_desc(x, x.Cp, s["wa"].shape[0], s["wc"].shape[0], s["kt"], s["sb"],
                                       s["ws"] is not None, s["act"])
        th, tw, tc, smem = C.c_int(), C.c_int(), C.c_int(), C.c_longlong()
        L.check(L.load().pv_bottleneck_fused_tiling(C.byref(d), 132, C.byref(th), C.byref(tw), C.byref(tc),
                                                    C.byref(smem)), "pv_bottleneck_fused_tiling")
        out.append((th.value, tw.value, tc.value))
    return out


def test_fused_block_tiling_pinned_per_swept_batch(slowfast_plans):
    got = {B: _fused_tilings(p) for B, p in slowfast_plans.items()}
    assert all(len(v) == 7 for v in got.values()), got
    assert got == FUSED_TILINGS, got
    assert len({tuple(v) for v in got.values()}) > 1
