"""Golden vectors of the MViT builder variants (norm="batchnorm" before / after fuse_bn(), pool_first, average pooling,
token input, headless, a stand-alone BatchNorm MultiScaleBlock) -> tests/golden/mvit_variants.pt.

For each entry of testing.MVIT_VARIANT_CASES: build this package's module and the reference's with the same builder
arguments, record the reference's ``state_dict`` keys, shapes and ``repr`` (this package's must equal them), load the
seeded weights into the reference (before fuse_bn(): both trees then run the same fuse_bn() on equal state), run the
reference's CPU forward on the seeded input and store the output with the seeds and checksums.  Also records the plan
``lower_only`` makes from the REFERENCE's own module tree.  Runs only where the reference package is importable: put its
checkout on PYTHONPATH.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_mvit_variants.py
"""
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "mvit_variants.pt")


def main():
    import pytorchvideo.models.vision_transformers as RV       # the reference
    import pytorchvideo.layers.attention as RA
    import pytorchvideo_b200.models.vision_transformers as PV   # this package's parameter containers
    import pytorchvideo_b200.layers.attention as PA
    from pytorchvideo_b200 import testing as TS
    from pytorchvideo_b200.engine.lower import lower_only
    out = {}
    for case, (what, kw, shape, fuse) in TS.MVIT_VARIANT_CASES.items():
        mine, x, extra = TS.build_mvit_variant_case(case, PV.create_multiscale_vision_transformers, PA.MultiScaleBlock)
        pre, _, _ = TS.build_mvit_variant_case(case, PV.create_multiscale_vision_transformers, PA.MultiScaleBlock,
                                               fuse=False)
        ref, _, _ = TS.build_mvit_variant_case(case, RV.create_multiscale_vision_transformers, RA.MultiScaleBlock,
                                               fuse=False)
        ref.load_state_dict(pre.state_dict(), strict=True)
        if fuse:
            ref.fuse_bn()
        sd = ref.state_dict()
        rec = {"keys": list(sd.keys()), "shapes": [list(v.shape) for v in sd.values()], "repr": repr(ref)}
        assert rec["keys"] == list(mine.state_dict().keys()), case
        assert rec["repr"] == repr(mine), case
        for k, v in mine.state_dict().items():
            assert torch.equal(v, sd[k]), (case, k)
        with torch.no_grad():
            y = ref(x.clone(), *extra)
        if isinstance(y, tuple):
            y, thw = y
            rec["thw"] = list(thw)
        plan, oshape = lower_only(ref, torch.zeros(x.shape), extra=tuple(tuple(e) for e in extra))
        rec.update({"weight_seed": 1234, "input_seed": 42, "output": y.clone(), "state_checksum": TS.state_checksum(mine),
                    "input_checksum": TS.tensor_checksum(x), "ref_ops": [n for n, _ in plan.ops],
                    "ref_stats": dict(plan.stats), "out_shape": list(oshape),
                    "batchnorms": sum(isinstance(m, (torch.nn.BatchNorm1d, torch.nn.BatchNorm3d)) for m in ref.modules())})
        out[case] = rec
        print("%-20s ok  out %s  |out|max %.4f  ops %d  BN %d" % (case, tuple(y.shape), float(y.abs().max()),
                                                                len(plan.ops), rec["batchnorms"]), flush=True)
    # the deprecation warning of create_scriptable_model with the BatchNorm model
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        RV.create_multiscale_vision_transformers(spatial_size=32, temporal_size=2, depth=1, norm="batchnorm",
                                                 create_scriptable_model=True)
    out["_scriptable_warning"] = [(c.category.__name__, str(c.message)) for c in w
                                  if issubclass(c.category, DeprecationWarning)]
    torch.save(out, GOLD)


if __name__ == "__main__":
    main()
