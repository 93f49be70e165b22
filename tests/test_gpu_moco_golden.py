"""GPU: MoCo v2, KnnMemory and ContrastiveLoss end to end against tests/golden/knn_moco.pt, the trainer's own
MOCOV2Module.training_step, KnnMemory and ContrastiveLoss run on the CPU (oracle/gen_golden_knn_moco.py).

- Bit-exact: the momentum parameters after every step (pv_ema_update), the queue rows the step did not write, ptr,
  the RNG state after every step (one randperm per view), the kNN memory after update sequences, the queue rows the
  step wrote equal the keys it computed, and the keys equal permute -> momentum plan -> unpermute.
- Losses, queue keys and embeddings: f32 within 2e-4 relative (+1e-5 absolute) for losses and 2e-4 absolute for unit
  rows; the f16 trunk within the tiers of test_gpu_ssl.py (3e-2 relative + 2e-3, and 3e-2).
- eval_knn preds within 2e-4 relative (NaN where the reference's are) on every query whose neighbour set equals the
  reference's; a query whose set differs may only differ at the k-th neighbour by a rounding-level similarity tie.
- The momentum plan is refreshed in place across steps, not compiled again (compile count).
"""
import hashlib
import os
import types

import pytest
import torch

from pytorchvideo_b200 import config, contrastive as K, testing as TS
from pytorchvideo_b200.losses import ContrastiveLoss
from pytorchvideo_b200.models.knn_memory import KnnMemory
from pytorchvideo_b200.models.moco_v2 import MOCO, MoCoQueue, create_mlp_util, create_moco_resnet_50
from pytorchvideo_b200.models.resnet import create_resnet

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "knn_moco.pt")
NS = types.SimpleNamespace(MOCO=MOCO, create_moco_resnet_50=create_moco_resnet_50, create_mlp_util=create_mlp_util,
                           create_resnet=create_resnet)
DEV = "cuda"
TIERS = {"f32": (2e-4, 1e-5, 2e-4), "f16": (3e-2, 2e-3, 3e-2)}


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def _ran(counts, *names):
    for n in names:
        assert counts.get(n, 0) >= 1, "%s did not run: %s" % (n, counts)


def _setup(name):
    model, views, k, dim = TS.build_moco_case(name, NS)
    knn = None
    if name == "moco_linear_v2":
        torch.manual_seed(TS.MOCO_QUEUE_SEED - 1)
        knn = KnnMemory(20, dim, momentum=0.5, knn_k=3)
        knn.memory = knn.memory.to(DEV)
    torch.manual_seed(TS.MOCO_QUEUE_SEED)
    queue = MoCoQueue(dim, k, batch_shuffle=True)
    return model.to(DEV), [v.to(DEV) for v in views], queue.to(DEV), knn


def _close_rows(got, want, tol):
    err = float((got.cpu() - want).abs().max())
    assert err <= tol, err
    return err


@pytest.mark.parametrize("precision", ["f32", "f16"])
@pytest.mark.parametrize("name", list(TS.MOCO_CASES))
def test_moco_step_vs_reference(gold, name, precision, monkeypatch):
    from pytorchvideo_b200.engine import lower as LW
    g = gold["moco"][name]
    rl, al, ae = TIERS[precision]
    config.set_precision(precision)
    try:
        model, views, queue, knn = _setup(name)
        small = isinstance(g["queue0"], torch.Tensor)
        if small:
            assert torch.equal(queue.queue_x.cpu(), g["queue0"])
        compiles = []
        real = LW.compile_model
        monkeypatch.setattr(LW, "compile_model", lambda *a, **k: compiles.append(1) or real(*a, **k))
        torch.manual_seed(TS.MOCO_STEP_SEED)
        loss = ContrastiveLoss()
        video_index = torch.tensor([3, 17, 3, 9], device=DEV)
        plan = None
        for i, gs in enumerate(g["steps"]):
            ptr0 = int(queue.ptr[0])
            before = queue.queue_x.clone()
            n0 = len(compiles)
            losses, counts = TS.launched_kernels(queue.step, model, views, loss, knn, video_index)
            _ran(counts, "ema_update_kernel", "refresh_gather_kernel", "l2_normalize_kernel<float>",
                 "bank_score_kernel<lse,32,vec4>", "queue_ce_rows_kernel", "bank_mean_kernel")
            (cm, refresh), = model._state()["plans"].values()
            assert refresh is not None
            if i == 0:
                plan = cm
            else:
                assert cm is plan and len(compiles) == n0, "the momentum plan was compiled again"
            assert torch.equal(torch.get_rng_state(), gs["rng"])
            assert int(queue.ptr[0]) == gs["ptr"]
            for p, want in zip(model.backbone_mmt.parameters(), gs["mmt_params"]):
                if small:
                    assert torch.equal(p.detach().cpu(), want)
                else:
                    assert hashlib.sha256(p.detach().cpu().numpy().tobytes()).hexdigest() == want
            V, B = len(views), views[0].shape[0]
            written = torch.zeros(queue.k, dtype=torch.bool)
            for v in range(V):
                written[(ptr0 + v * B) % queue.k:(ptr0 + v * B) % queue.k + B] = True
            assert torch.equal(queue.queue_x.cpu()[~written], before.cpu()[~written])
            # the keys the step wrote are the momentum embeddings of its views, after its momentum update
            keys = torch.cat([model.forward_backbone_mmt(x) for x in views])
            idx = torch.cat([torch.arange(ptr0 + v * B, ptr0 + (v + 1) * B) % queue.k for v in range(V)])
            assert torch.equal(queue.queue_x[idx.to(DEV)], keys)
            if small:
                _close_rows(queue.queue_x, gs["queue"], ae)
            else:
                got = TS.tensor_checksum(queue.queue_x)
                assert abs(got[0] - gs["queue"][0]) <= ae * len(idx) * queue.dim
                assert abs(got[2] - gs["queue"][2]) <= 2 * ae * len(idx) * queue.dim
            for a, b in zip(losses, gs["losses"]):
                assert a.dim() == 0
                err = abs(float(a) - b)
                print("RATIO moco %s %s step %d loss_err %.3e (%.3f)" % (name, precision, i, err, err / (rl * abs(b) + al)))
                assert err <= rl * abs(b) + al
        _close_rows(model(views[0]), g["embedding"], ae)
        _close_rows(model.forward_backbone_mmt(views[0]), g["embedding_mmt"], ae)
        if knn is not None:
            _close_rows(knn.memory, g["knn_memory"], 1e-6 if precision == "f32" else ae)
    finally:
        config.set_precision("f16")


@pytest.mark.parametrize("name", ["moco_linear_v3", "moco_slow_r50"])
def test_moco_keys_equal_permute_plan_unpermute(name):
    model, views, queue, _ = _setup(name)
    torch.manual_seed(1)
    keys, counts = TS.launched_kernels(queue.compute_keys, model, views)
    _ran(counts, "l2_normalize_kernel<float>")
    g = torch.Generator().manual_seed(1)
    for v, x in enumerate(views):
        perm = torch.randperm(x.shape[0], generator=g).to(DEV)
        shuffled = model.forward_backbone_mmt(x[perm])
        restore = torch.argsort(perm)
        assert torch.equal(shuffled[restore], keys[v])


@pytest.mark.parametrize("name", list(TS.KNN_UPDATES))
def test_knn_update_sequences_bit_exact(gold, name):
    g = gold["knn_update"][name]
    M, dim, mmt, _ = TS.KNN_UPDATES[name]
    knn = KnnMemory(M, dim, momentum=mmt)
    knn.memory = g["before"].clone().to(DEV)
    for (x, ind), want in zip(TS.knn_update_inputs(name), g["after"]):
        _, counts = TS.launched_kernels(knn.update, x.to(DEV), ind.to(DEV))
        _ran(counts, "bank_update_kernel")
        assert torch.equal(knn.memory.cpu(), want)


def _check_preds(name, got_preds, got_idx, gp, gi, sims):
    agree = 0
    for n in range(gp.shape[0]):
        if set(got_idx[n].tolist()) == set(gi[n].tolist()):
            agree += 1
            a, b = got_preds[n].double(), gp[n].double()
            assert torch.equal(torch.isnan(a), torch.isnan(b)), n
            fin = torch.isfinite(b)
            assert torch.equal(a[~fin & ~torch.isnan(b)], b[~fin & ~torch.isnan(b)])
            assert bool(((a[fin] - b[fin]).abs() <= 2e-4 * b[fin].abs() + 1e-30).all()), n
        else:                      # only the boundary neighbour may differ, by a similarity tie at rounding level
            diff = set(got_idx[n].tolist()) ^ set(gi[n].tolist())
            assert len(diff) == 2, (n, diff)
            s = sims[n][list(diff)]
            assert float((s[0] - s[1]).abs()) <= 1e-5, (n, s)
    print("KNN %s: %d of %d queries with the reference's neighbour set" % (name, agree, gp.shape[0]))
    assert agree >= gp.shape[0] - max(1, gp.shape[0] // 16)


@pytest.mark.parametrize("name", list(TS.KNN_CASES))
def test_eval_knn_vs_reference(gold, name):
    g = gold["knn"][name]
    knn, q = TS.knn_case(name, KnnMemory)
    assert TS.tree_digests(knn) == g["tree"]
    knn.memory = knn.memory.to(DEV)
    knn.train_labels = knn.train_labels.to(DEV)
    preds, counts = TS.launched_kernels(knn.eval_knn, q.to(DEV))
    _ran(counts, "bank_merge_vote_kernel")
    _, idx, _ = K.bank_topk(q.to(DEV), knn.memory, knn.knn_k, knn.train_labels, knn.downstream_classes,
                            knn.temperature)
    sims = (q.double() @ knn.memory.cpu().double().T)
    _check_preds(name, preds.cpu(), idx.cpu(), g["preds"], g["idx"], sims)


def test_eval_knn_overflow_vs_reference(gold):
    g = gold["knn"]["overflow"]
    knn, q, x, ind = TS.knn_overflow_case(KnnMemory)
    knn.memory = knn.memory.to(DEV)
    knn.train_labels = knn.train_labels.to(DEV)
    _, counts = TS.launched_kernels(knn.update, x.to(DEV), ind.to(DEV))
    _ran(counts, "bank_update_kernel")
    preds, counts = TS.launched_kernels(knn.eval_knn, q.to(DEV))
    _ran(counts, "bank_score_kernel<topk,32,vec4>", "bank_merge_vote_kernel")
    assert bool(torch.isnan(g["preds"]).any())
    assert torch.allclose(preds.cpu(), g["preds"], rtol=2e-4, atol=0, equal_nan=True)


@pytest.mark.parametrize("reduction", ["mean", "none"])
def test_contrastive_loss_vs_reference(gold, reduction):
    x, want = gold["contrastive_loss"][reduction]
    got, counts = TS.launched_kernels(ContrastiveLoss(reduction, 0.1), x.to(DEV))
    _ran(counts, "logits_ce_rows_kernel")
    assert got.shape == want.shape
    assert bool(((got.cpu() - want).abs() <= 2e-4 * want.abs() + 1e-5).all())
