"""Golden vectors of the Efficient X3D cases (testing.EFFICIENT_CASES) -> tests/golden/efficient_x3d.pt.

For every case: build this package's module and the reference's with the same arguments, check that their state_dict
keys and ``repr`` agree, copy the weights with ``load_state_dict(strict=True)``, run the reference's CPU forward and pin
``efficient_forward`` (oracle/efficient_ref.py) to it bit for bit on both module trees.  Records the output, the seed,
the state / input checksums, digests of the ``repr`` and ``state_dict`` keys and (by its digest, under "launch_lists") the ``lower_only`` launch list of the REFERENCE's own module tree (the lowering
dispatches on class names); no weights.  Also checks that the reference's deployable form (its own
``convert_to_deployable_form``) is refused by the lowering.  Runs only where the reference package is importable: put
its checkout on PYTHONPATH.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_efficient.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "efficient_x3d.pt")
SEED = 31


def main():
    from pytorchvideo_b200 import testing as TS
    from pytorchvideo_b200.engine.lower import lower_only
    from oracle.efficient_ref import efficient_forward
    mine_ns, ref_ns = TS.efficient_namespace(), TS.efficient_namespace("pytorchvideo")
    out, lists = {}, {}
    for case in TS.EFFICIENT_CASES:
        mine, x = TS.build_efficient_case(case, mine_ns, seed=SEED)
        ref, _ = TS.build_efficient_case(case, ref_ns, seed=SEED)
        assert list(ref.state_dict().keys()) == list(mine.state_dict().keys()), case
        assert repr(ref) == repr(mine), case
        ref.load_state_dict(mine.state_dict(), strict=True)
        with torch.no_grad():
            y = ref(x.clone())
        assert torch.equal(efficient_forward(ref, x), y), "oracle != reference on reference modules (%s)" % case
        assert torch.equal(efficient_forward(mine, x), y), "oracle != reference on product tree (%s)" % case
        plan, _ = lower_only(ref, x)
        launches = [(md["name"], md["kind"]) for md in plan.meta]
        lid = TS.tree_digests_text(repr(launches))
        lists.setdefault(lid, launches)       # the model cases share two lists: each is stored once
        out[case] = {"seed": SEED, "output": y.clone(), "state_checksum": TS.state_checksum(mine),
                     "input_checksum": TS.tensor_checksum(x), "tree_digests": TS.tree_digests(ref),
                     "launches": lid}
        print("%-22s ok  out %s  |out|max %.4f  launches %d" % (case, tuple(y.shape), float(y.abs().max()),
                                                               len(plan.meta)), flush=True)
    # the reference's deployable form: Conv2d decompositions the lowering refuses, naming the first module
    from pytorchvideo.accelerator.deployment.mobile_cpu.utils.model_conversion import convert_to_deployable_form
    ref, x = TS.build_efficient_case("xs_no_head", ref_ns, seed=SEED)
    dep = convert_to_deployable_form(ref, x)
    try:
        lower_only(dep, x)
    except NotImplementedError as e:
        assert "s1.pathway0_stem_conv_xy" in str(e), e
    else:
        raise AssertionError("the deployable form was lowered")
    out["launch_lists"] = lists
    torch.save(out, GOLD)


if __name__ == "__main__":
    main()
