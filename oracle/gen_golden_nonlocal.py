"""Golden vectors of the Non-local block cases (testing.NONLOCAL_CASES) -> tests/golden/nonlocal.pt.

For every case: build this package's ``create_nonlocal`` module and the reference's with the same arguments, check
that their state_dict keys and ``repr`` agree, copy the weights with ``load_state_dict(strict=True)``, run the
reference's CPU forward, and pin ``nonlocal_forward`` (oracle/nonlocal_ref.py, on both module trees) to it bit for bit.  Writes the outputs,
the seeds and the state / input checksums; no weights (the tests rebuild them from the seed).  Runs only where the
reference package is importable: put its checkout on PYTHONPATH.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_nonlocal.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "nonlocal.pt")
SEED = 91


def main():
    from pytorchvideo.layers.nonlocal_net import create_nonlocal as ref_create       # the reference
    from pytorchvideo_b200.layers.nonlocal_net import create_nonlocal
    from pytorchvideo_b200 import testing as TS
    from oracle.nonlocal_ref import nonlocal_forward
    out = {}
    for case in TS.NONLOCAL_CASES:
        mine, x = TS.build_nonlocal_case(case, create_nonlocal, seed=SEED)
        kw, shape = TS.NONLOCAL_CASES[case]
        ref = ref_create(**kw).eval()
        assert list(ref.state_dict().keys()) == list(mine.state_dict().keys()), case
        assert repr(ref) == repr(mine), case
        ref.load_state_dict(mine.state_dict(), strict=True)
        with torch.no_grad():
            y = ref(x.clone())
        assert torch.equal(nonlocal_forward(ref, x), y), "oracle != reference on reference modules (%s)" % case
        assert torch.equal(nonlocal_forward(mine, x), y), "oracle != reference on product tree (%s)" % case
        out[case] = {"kwargs": {k: v for k, v in kw.items() if k != "norm"}, "norm": "none" if "norm" in kw else "bn",
                     "shape": tuple(shape), "seed": SEED, "output": y.clone(),
                     "input_checksum": TS.tensor_checksum(x), "state_checksum": TS.state_checksum(mine)}
        print("%-28s ok  out %s  |out|max %.4f" % (case, tuple(y.shape), float(y.abs().max())), flush=True)
    torch.save(out, GOLD)


if __name__ == "__main__":
    main()
