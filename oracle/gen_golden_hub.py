"""Golden vectors of the image MViT-B-16 and SlowFast-16x8-R101-50-50 hub entries -> tests/golden/hub_tail.pt.

For each entry of testing.HUB_TAIL_CASES: build this package's model and the reference's hub model, record the
reference's ``state_dict`` keys, shapes and ``repr`` (this package's must equal them), copy the seeded weights into the
reference with ``load_state_dict(strict=True)``, run the reference's CPU forward on the seeded input and store the
logits with the seeds and checksums (the inputs are regenerated from their seeds; no weights are stored).  Also
records the plan ``lower_only`` makes from the REFERENCE's own module tree (op names and kernel counts: the lowering
dispatches on class and attribute names, so the same plan means the same logits) and, for the image MViT, the
multiply-accumulates of one image counted with forward hooks on the reference (Conv2d / Conv3d:
out.numel * Cin/groups * taps; Linear: out.numel * in_features; attention: 2 * B * Nq * Nk * dim).  Runs only where
the reference package is importable: put its checkout on PYTHONPATH.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_hub.py
"""
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "hub_tail.pt")


def hook_macs(model, x):
    """Multiply-accumulates of one forward, counted with hooks (see the module docstring)."""
    total, hooks, pooled_k = [0], [], {}

    def conv_hook(m, inp, out):
        total[0] += out.numel() * (m.in_channels // m.groups) * m.weight[0, 0].numel()

    def linear_hook(m, inp, out):
        total[0] += out.numel() * m.in_features

    def attn_hook(m, inp, out):
        xin, y = inp[0], out[0]
        nk = pooled_k.get(id(m), xin.shape[1])
        total[0] += 2 * y.shape[0] * y.shape[1] * nk * m.dim_out if hasattr(m, "dim_out") else 0

    for m in model.modules():
        if isinstance(m, (nn.Conv2d, nn.Conv3d)):
            hooks.append(m.register_forward_hook(conv_hook))
        elif isinstance(m, nn.Linear):
            hooks.append(m.register_forward_hook(linear_hook))
        elif type(m).__name__ == "MultiScaleAttention":
            hooks.append(m.register_forward_hook(attn_hook))
            if getattr(m, "pool_k", None) is not None:
                def k_hook(pm, inp, out, owner=m):
                    pooled_k[id(owner)] = 1 + out[0, 0].numel() if owner.has_cls_embed else out[0, 0].numel()
                hooks.append(m.pool_k.register_forward_hook(k_hook))
    with torch.no_grad():
        model(x)
    for h in hooks:
        h.remove()
    return total[0]


def main():
    import pytorchvideo.models.hub as RH            # the reference
    import pytorchvideo_b200.models.hub as PH       # this package's parameter containers
    from pytorchvideo_b200 import testing as TS
    from pytorchvideo_b200.engine.lower import lower_only
    out = {}
    for case in TS.HUB_TAIL_CASES:
        mine, x = TS.build_hub_tail_case(case, PH, weight_seed=1234, input_seed=42)
        ref = getattr(RH, case)(pretrained=False).eval()
        sd = ref.state_dict()
        rec = {"keys": list(sd.keys()), "shapes": [list(v.shape) for v in sd.values()], "repr": repr(ref)}
        assert rec["keys"] == list(mine.state_dict().keys()) and rec["repr"] == repr(mine), case
        ref.load_state_dict(mine.state_dict(), strict=True)
        with torch.no_grad():
            y = ref(list(x) if isinstance(x, list) else x.clone())
        plan, shape = lower_only(ref, [torch.zeros(t.shape) for t in x] if isinstance(x, list) else torch.zeros(x.shape))
        rec.update({"weight_seed": 1234, "input_seed": 42, "output": y.clone(), "state_checksum": TS.state_checksum(mine),
                    "input_checksum": [TS.tensor_checksum(t) for t in x] if isinstance(x, list) else TS.tensor_checksum(x),
                    "ref_ops": [n for n, _ in plan.ops], "ref_stats": dict(plan.stats), "out_shape": list(shape)})
        if case == "mvit_base_16":
            rec["ref_macs_per_image"] = hook_macs(ref, x[:1])
        out[case] = rec
        print("%-26s ok  out %s  |out|max %.4f  ops %d" % (case, tuple(y.shape), float(y.abs().max()), len(plan.ops)),
              flush=True)
    torch.save(out, GOLD)


if __name__ == "__main__":
    main()
