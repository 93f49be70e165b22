"""Golden vectors of the self-supervised models, the projector builder and the soft-target loss (tests/golden/ssl.pt).

Runs the reference's own SimCLR, BYOL, MemoryBank, make_multilayer_perceptron and SoftTargetCrossEntropyLoss on the
CPU (eval mode) for every testing.SSL_CASES / SOFT_CE_CASES entry: the reference unit-test configurations and a
Slow-R50 trunk (head projection removed) with a [2048, 2048, 128] BatchNorm projector on 8 x 224^2 clips.  Weights and
inputs are regenerated from seeds by the tests; the file holds the losses, the normalised embeddings, BYOL's momentum
parameters after the call (checksums), MemoryBank's bank checksum and its drawn indices, and the tree digests.  Runs
only where the reference package is importable: put its checkout on PYTHONPATH.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_ssl.py
"""
import hashlib
import os
import sys
import types

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "ssl.pt")
FORWARD_SEED = 77              # torch.manual_seed before every forward (MemoryBank draws its indices there)


def reference_namespace():
    from pytorchvideo.layers.mlp import make_multilayer_perceptron
    from pytorchvideo.models.byol import BYOL
    from pytorchvideo.models.memory_bank import MemoryBank
    from pytorchvideo.models.resnet import create_resnet
    from pytorchvideo.models import simclr
    from pytorchvideo.models.simclr import SimCLR
    # oracle/shim's differentiable_all_gather raises NotImplementedError (it stands in for a training-only
    # collective); fvcore's own returns [input] in a single process, which is restated here
    simclr.differentiable_all_gather = lambda t: [t]
    return types.SimpleNamespace(SimCLR=SimCLR, BYOL=BYOL, MemoryBank=MemoryBank, create_resnet=create_resnet,
                                 make_multilayer_perceptron=make_multilayer_perceptron)


@torch.no_grad()
def run_case(name, ns):
    from pytorchvideo_b200 import testing as TS
    m, args = TS.build_ssl_case(name, ns)
    out = {"tree": TS.tree_digests(m)}
    if name.startswith("simclr"):
        emb = F.normalize(m.mlp(m.backbone(args[0]) if m.backbone is not None else args[0]), p=2, dim=1)
        out["embedding"] = emb
    elif name.startswith("byol"):
        out["embedding"] = m.forward_backbone(args[0])
        out["embedding_mmt_before"] = m.forward_backbone_mmt(args[0])
    else:
        out["memory"] = TS.tensor_checksum(m.memory)
        out["embedding"] = F.normalize(m.mlp(m.backbone(args[0])) if m.mlp is not None else m.backbone(args[0]),
                                       p=2, dim=1)
        torch.manual_seed(FORWARD_SEED)
        out["indices"] = torch.randint(0, m.bank_size, size=(args[0].shape[0], m.neg_size + 1))
        out["indices"].select(1, 0).copy_(args[1])
    torch.manual_seed(FORWARD_SEED)
    out["loss"] = float(m(*args))
    if name.startswith("byol"):
        out["mmt_params"] = [hashlib.sha256(p.detach().numpy().tobytes()).hexdigest() for p in m.backbone_mmt.parameters()]
        out["mmt_param_values"] = [p.detach().clone() for p in m.backbone_mmt.parameters()] if not name.endswith(
            "_video") else None
        out["embedding_mmt_after"] = m.forward_backbone_mmt(args[0])
    print("%-20s loss %.6f" % (name, out["loss"]))
    return out


def main():
    from pytorchvideo.losses.soft_target_cross_entropy import SoftTargetCrossEntropyLoss
    from pytorchvideo.layers.mlp import make_multilayer_perceptron
    from pytorchvideo_b200 import testing as TS
    ns = reference_namespace()
    gold = {"cases": {n: run_case(n, ns) for n in TS.SSL_CASES}, "soft_ce": {}, "mlp": {}}
    for n in TS.SOFT_CE_CASES:
        x, t, kw = TS.soft_ce_case(n)
        gold["soft_ce"][n] = SoftTargetCrossEntropyLoss(**kw)(x, t)
    for dims, kw in (([8, 4, 2], {}), ([2048, 2048, 128], {"norm": torch.nn.BatchNorm1d}),
                     ([16, 0, 4], {"dropout_rate": 0.5, "final_activation": None})):
        mlp, od = make_multilayer_perceptron(dims, **kw)
        gold["mlp"][str(dims)] = {"repr": repr(mlp), "keys": list(mlp.state_dict()), "output_dim": od}
    torch.save(gold, GOLD)
    print("wrote", GOLD)


if __name__ == "__main__":
    main()
