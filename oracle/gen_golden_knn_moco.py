"""Golden vectors of the kNN memory, the contrastive loss and MoCo v2 (tests/golden/knn_moco.pt).

Loads the trainer's own module/ssl_helper.py, module/losses.py and module/moco_v2.py by file path (the trainer
package's __init__ needs Lightning): hydra, omegaconf, torchrecipes, pytorch_lightning and the video_classification
module get stubs, and module/distributed_utils.py is loaded by path too.  Then, on the CPU and in eval mode:
- MoCo: the reference's own MOCOV2Module.__init__ (queue draw) and training_step on every testing.MOCO_CASES entry,
  with manual_backward and log stubbed to capture the per-view losses: losses, queue checksum / contents and ptr after
  every step (the linear cases wrap the queue), the momentum parameters, the RNG state after each step, the online
  and momentum embeddings after the steps, the kNN memory the linear V = 2 case updates, and tree digests.
- KnnMemory.eval_knn preds for every testing.KNN_CASES entry and the overflow case (with the neighbour indices, so a
  test can tell a rounding-level reordering at the k-th neighbour from an error), and the bank after every
  testing.KNN_UPDATES sequence.  Updates run on one thread: there the CPU index_put_ keeps the last occurrence of a
  repeated index (with several threads, occurrences in different chunks race).
Runs only where the reference checkout exists (REFERENCE, default /root/reference).

    python oracle/gen_golden_knn_moco.py
"""
import dataclasses
import hashlib
import importlib.util
import os
import sys
import types

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
sys.path.insert(1, REF)

GOLD = os.path.join(ROOT, "tests", "golden", "knn_moco.pt")
MODULE_DIR = os.path.join(REF, "pytorchvideo_trainer", "pytorchvideo_trainer", "module")


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__path__ = []
    sys.modules[name] = m
    return m


def _load(name, fname):
    spec = importlib.util.spec_from_file_location(name, os.path.join(MODULE_DIR, fname))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


class _VideoClassificationModule(nn.Module):
    """Stands in for the Lightning base: keeps model and loss, and the manual-optimisation hooks capture."""

    def __init__(self, model, loss, modality_key="video", **kw):
        super().__init__()
        self.model = model
        self.loss = loss
        self.modality_key = modality_key
        self.captured = []

    @property
    def device(self):
        return torch.device("cpu")

    def manual_zero_opt_grad(self):
        pass

    def manual_update_lr(self):
        pass

    def manual_opt_step(self):
        pass

    def manual_backward(self, loss):
        self.captured.append(float(loss))

    def log(self, *a, **k):
        pass


def reference_modules():
    @dataclasses.dataclass
    class ModuleConf:
        pass

    class ConfigStore:
        def store(self, **kw):
            pass

    _stub("hydra", utils=types.SimpleNamespace(instantiate=lambda c: c))
    _stub("hydra.utils", instantiate=lambda c: c)
    _stub("hydra.core")
    _stub("hydra.core.config_store", ConfigStore=ConfigStore)
    _stub("omegaconf", MISSING="???")
    _stub("torchrecipes")
    _stub("torchrecipes.core")
    _stub("torchrecipes.core.conf", ModuleConf=ModuleConf)
    _stub("torchrecipes.utils")
    _stub("torchrecipes.utils.config_utils", get_class_name_str=lambda c: c.__name__)
    _stub("pytorch_lightning")
    _stub("pytorch_lightning.trainer", Trainer=object)
    _stub("pytorchvideo_trainer")
    _stub("pytorchvideo_trainer.module")
    _stub("pytorchvideo_trainer.module.video_classification", Batch=dict, BatchKey=str, EnsembleMethod=str,
          VideoClassificationModule=_VideoClassificationModule)
    _load("pytorchvideo_trainer.module.distributed_utils", "distributed_utils.py")
    ssl = _load("pytorchvideo_trainer.module.ssl_helper", "ssl_helper.py")
    losses = _load("pytorchvideo_trainer.module.losses", "losses.py")
    moco = _load("pytorchvideo_trainer.module.moco_v2", "moco_v2.py")
    return ssl, losses, moco


def sha(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


@torch.no_grad()
def run_moco(name, ssl, losses, moco):
    from pytorchvideo.models.resnet import create_resnet
    from pytorchvideo_b200 import testing as TS
    ns = types.SimpleNamespace(MOCO=moco.MOCO, create_moco_resnet_50=moco.create_moco_resnet_50,
                               create_mlp_util=ssl.create_mlp_util, create_resnet=create_resnet)
    model, views, k, dim = TS.build_moco_case(name, ns)
    knn = None
    if name == "moco_linear_v2":
        torch.manual_seed(TS.MOCO_QUEUE_SEED - 1)
        knn = ssl.KnnMemory(20, dim, momentum=0.5, knn_k=3)
    torch.manual_seed(TS.MOCO_QUEUE_SEED)
    mod = moco.MOCOV2Module(model=model, loss=losses.ContrastiveLoss(), optim=None, metrics=[], dim=dim, k=k,
                            batch_shuffle=True, local_shuffle_bn=False, knn_memory=knn)
    mod.trainer = types.SimpleNamespace(world_size=1, current_epoch=1, max_epochs=1, num_gpus=1)
    mod.cur_epoch_step = 0
    mod.no_update_iters = 0
    mod.eval()
    small = k * dim <= 4096
    out = {"tree": TS.tree_digests(model), "module_keys": list(mod.state_dict()),
           "queue0": mod.queue_x.clone() if small else TS.tensor_checksum(mod.queue_x), "steps": []}
    torch.manual_seed(TS.MOCO_STEP_SEED)
    video_index = torch.tensor([3, 17, 3, 9])
    for _ in range(TS.MOCO_STEPS[name]):
        mod.captured = []
        mod.training_step({"video": views, "video_index": video_index}, 0)
        out["steps"].append({
            "losses": list(mod.captured),
            "ptr": int(mod.ptr[0]),
            "queue": mod.queue_x.clone() if small else TS.tensor_checksum(mod.queue_x),
            "rng": torch.get_rng_state().clone(),
            "mmt_params": [p.detach().clone() for p in model.backbone_mmt.parameters()] if small else
            [sha(p) for p in model.backbone_mmt.parameters()],
        })
        print("%-16s ptr %2d losses %s" % (name, out["steps"][-1]["ptr"], out["steps"][-1]["losses"]))
    out["embedding"] = model(views[0])
    out["embedding_mmt"] = model.forward_backbone_mmt(views[0])
    if knn is not None:
        out["knn_memory"] = knn.memory.clone()
    return out


@torch.no_grad()
def main():
    from pytorchvideo_b200 import testing as TS
    ssl, losses, moco = reference_modules()
    gold = {"moco": {}, "knn": {}, "knn_update": {}}
    threads = torch.get_num_threads()
    torch.set_num_threads(1)                  # index_put_ keeps the last of repeated indices on one thread
    try:
        for name in TS.MOCO_CASES:
            gold["moco"][name] = run_moco(name, ssl, losses, moco)
        for name in TS.KNN_UPDATES:
            M, dim, mmt, _ = TS.KNN_UPDATES[name]
            torch.manual_seed(61)
            knn = ssl.KnnMemory(M, dim, momentum=mmt)
            gold["knn_update"][name] = {"before": knn.memory.clone(), "after": []}
            for x, ind in TS.knn_update_inputs(name):
                knn.update(x, ind)
                gold["knn_update"][name]["after"].append(knn.memory.clone())
        torch.set_num_threads(threads)
        for name in TS.KNN_CASES:
            knn, q = TS.knn_case(name, ssl.KnnMemory)
            dist = q @ knn.memory.T
            _, yi = dist.topk(knn.knn_k, dim=1, largest=True, sorted=True)
            gold["knn"][name] = {"preds": knn.eval_knn(q), "idx": yi, "tree": TS.tree_digests(knn)}
        knn, q, x, ind = TS.knn_overflow_case(ssl.KnnMemory)
        knn.update(x, ind)
        dist = q @ knn.memory.T
        _, yi = dist.topk(knn.knn_k, dim=1, largest=True, sorted=True)
        gold["knn"]["overflow"] = {"preds": knn.eval_knn(q), "idx": yi}
        print("overflow row NaN count", int(torch.isnan(gold["knn"]["overflow"]["preds"]).sum()))
        gold["contrastive_loss"] = {}
        g = torch.Generator().manual_seed(71)
        for red in ("mean", "none"):
            x = torch.rand((6, 33), generator=g) * 2 - 1
            gold["contrastive_loss"][red] = (x, losses.ContrastiveLoss(red, 0.1)(x))
        gold["mlp"] = {"repr": repr(ssl.create_mlp_util(12, 8, 32, 3, norm=nn.BatchNorm1d)),
                       "xavier": [getattr(m, "xavier_init", None) for m in
                                  ssl.create_mlp_util(12, 8, 32, 3, norm=None)]}
    finally:
        torch.set_num_threads(threads)
    torch.save(gold, GOLD)
    print("wrote", GOLD, os.path.getsize(GOLD), "bytes")


if __name__ == "__main__":
    main()
