"""Golden vectors of the masked multistream cases (testing.MASKED_CASES) -> tests/golden/masked.pt.

For every case: build this package's module tree and the reference's with the same seeds, check that their state_dict
keys and ``repr`` agree, copy the weights with ``load_state_dict(strict=True)``, and run the reference's CPU forward on
clones of the inputs (the reference writes into its mask and, for max pooling, into x), and pin ``masked_forward``
(oracle/masked_ref.py, on both module trees, in float32 and float64) to it: bit for bit where it repeats the
reference's own ops, within ORACLE_TOL where the reference goes through MKL.  Writes the outputs, the
attention weights of every TransposeMultiheadAttention, the reprs and keys, the launch list the reference's own
tree lowers to, the seeds and the state / input checksums;
no weights (the tests rebuild them from the seed).  Runs only where the reference package is importable: put its
checkout on PYTHONPATH.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_masked.py
"""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "masked.pt")
SEED = 1234
# the oracle repeats the reference's own torch ops for these cases: bit-exact in float32
EXACT = ("pool_max", "pool_avg", "pool_sum", "pool_avg_nomask", "pool_max_t1", "default", "posenc")
# elsewhere the reference goes through MKL GEMMs, fused attention softmax and cuDNN-free packed LSTM steps: max |err|
# relative to max |output| (and absolute on the attention weights)
ORACLE_TOL = 2e-6


def namespaces():
    import pytorchvideo.models.masked_multistream as RM
    import pytorchvideo.layers.fusion as RF
    import pytorchvideo.layers.positional_encoding as RP
    import pytorchvideo_b200.models as MM
    import pytorchvideo_b200.layers as ML
    names = ("MaskedTemporalPooling", "LearnMaskedDefault", "TransposeMultiheadAttention", "TransposeTransformerEncoder",
             "LSTM", "MaskedSequential", "MaskedMultiPathWay")
    ref = types.SimpleNamespace(make_fusion_layer=RF.make_fusion_layer, PositionalEncoding=RP.PositionalEncoding,
                                **{n: getattr(RM, n) for n in names})
    mine = types.SimpleNamespace(make_fusion_layer=ML.make_fusion_layer, PositionalEncoding=ML.PositionalEncoding,
                                 **{n: getattr(MM, n) for n in names})
    return ref, mine


def main():
    from pytorchvideo_b200 import testing as TS
    from oracle.masked_ref import masked_forward
    from pytorchvideo_b200.engine.lower import lower_only
    ref_ns, my_ns = namespaces()
    out = {}
    for case in TS.MASKED_CASES:
        mine = TS.build_masked_case(case, my_ns, seed=SEED)
        ref = TS.build_masked_case(case, ref_ns, seed=SEED)
        assert list(ref.state_dict().keys()) == list(mine.state_dict().keys()), case
        assert repr(ref) == repr(mine), case
        ref.load_state_dict(mine.state_dict(), strict=True)
        x, mask = TS.masked_case_inputs(case)
        with torch.no_grad():
            y = TS.masked_call(ref, x.clone(), None if mask is None else mask.clone())
        weights = {n: mod.attention_weights.clone() for n, mod in ref.named_modules()
                   if type(mod).__name__ == "TransposeMultiheadAttention"}
        for tree in (ref, mine):            # the oracle, on both module trees
            o32, w32 = masked_forward(tree, x, mask)
            o64, w64 = masked_forward(tree, x, mask, torch.float64)
            if case in EXACT:
                assert torch.equal(o32, y), "oracle != reference (%s)" % case
            else:
                assert float((o32 - y).abs().max()) <= ORACLE_TOL * float(y.abs().max()), case
            assert float((o64 - y.double()).abs().max()) <= ORACLE_TOL * float(y.abs().max()), case
            assert sorted(w32) == sorted(weights), case
            for n, w in weights.items():
                assert float((w32[n] - w).abs().max()) <= ORACLE_TOL and float((w64[n] - w.double()).abs().max()) <= ORACLE_TOL
        ins, extra = TS.masked_engine_args(case, x, mask)
        launches = [op["name"] for op in lower_only(ref, ins, extra=extra)[0].meta]      # the reference's own tree
        out[case] = {"seed": SEED, "output": y.clone(), "weights": weights, "repr": repr(mine), "ref_launches": launches,
                     "keys": list(mine.state_dict().keys()), "input_checksum": TS.tensor_checksum(x),
                     "state_checksum": TS.state_checksum(mine)}
        print("%-24s ok  out %s  |out|max %.4f" % (case, tuple(y.shape), float(y.abs().max())), flush=True)
    torch.save(out, GOLD)


if __name__ == "__main__":
    main()
