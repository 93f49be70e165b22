"""Golden vectors of the grouped-convolution model cases (testing.GROUPED_MODEL_CASES).

Same recipe as the model loop of gen_golden.py: build each case with this repo's builders and with the reference's
hub builder (same kwargs), copy the weights with ``load_state_dict(strict=True)``, run the reference CPU forward, pin
``oracle_forward`` to it bit for bit, and write tests/golden/model_grouped_<case>.pt.  Runs only where the reference
is importable.

    python oracle/gen_golden_grouped.py [--only case]
"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
sys.path.insert(1, "/root/reference")

GOLD = os.path.join(ROOT, "tests", "golden")


def gen_grouped_models(only=None):
    import pytorchvideo.models.hub as RH            # the reference
    import pytorchvideo_b200.models.hub as PH       # this repo's parameter containers
    from pytorchvideo_b200 import testing as TS
    from oracle.interp import oracle_forward
    for case, (hub, kw, B, T, H, W, is_sf, grid) in TS.GROUPED_MODEL_CASES.items():
        if only and case != only:
            continue
        t0 = time.time()
        mine, inp, _ = TS.build_grouped_case(case, PH, weight_seed=1234, input_seed=42)
        ref = getattr(RH, hub)(pretrained=False, **kw)
        ref.load_state_dict(mine.state_dict(), strict=True)
        ref.eval()
        clip = TS.synthetic_clip(B, T, H, W, seed=42, f16_values=grid)
        with torch.no_grad():
            out_ref = ref(list(inp) if is_sf else inp)          # list() - the reference mutates it
            inp = TS.slowfast_inputs(clip) if is_sf else clip
            out_orc_on_mine = oracle_forward(mine, inp)
            out_orc_on_ref = oracle_forward(ref, inp)
        assert torch.equal(out_ref, out_orc_on_ref), "oracle != reference on reference modules (%s)" % case
        assert torch.equal(out_ref, out_orc_on_mine), "oracle != reference on product tree (%s)" % case
        torch.save({"case": case, "hub": hub, "kwargs": kw, "batch": B, "T": T, "H": H, "W": W, "weight_seed": 1234,
                    "input_seed": 42, "f16_grid": grid, "output": out_ref.clone(),
                    "input_checksum": TS.tensor_checksum(clip), "state_checksum": TS.state_checksum(mine)},
                   os.path.join(GOLD, "model_grouped_%s.pt" % case))
        print("%-18s ok  out %s  |out|max %.4f  (%.1fs)" % (case, tuple(out_ref.shape), float(out_ref.abs().max()),
                                                            time.time() - t0), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    gen_grouped_models(a.only)
