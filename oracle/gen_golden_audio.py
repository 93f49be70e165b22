"""Golden vectors of the audio cases (testing.AUDIO_CASES) -> tests/golden/audio.pt.

For every case: build this package's model and the reference's with the same arguments, check that their state_dict
keys and ``repr`` agree, copy the weights with ``load_state_dict(strict=True)``, run the reference's CPU forward
(its FuseAudioToFastSlow prints a debug size; that output is swallowed) and pin ``audio_forward`` (oracle/audio_ref.py)
to it bit for bit on both module trees.  Records the output, the seed, the state /
input checksums and the ``lower_only`` launch list of the REFERENCE's own module tree (the lowering dispatches on
class names); no weights.  Runs only where the reference package is importable: put its checkout on PYTHONPATH.

    PYTHONPATH=<reference checkout> python oracle/gen_golden_audio.py
"""
import contextlib
import io
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))

GOLD = os.path.join(ROOT, "tests", "golden", "audio.pt")
SEED = 2024


class _RefBuilders:
    from pytorchvideo.models.audio_visual_slowfast import create_audio_visual_slowfast      # the reference
    from pytorchvideo.models.resnet import create_acoustic_bottleneck_block, create_acoustic_resnet


def main():
    import pytorchvideo_b200.models as mine_builders
    from pytorchvideo_b200 import testing as TS
    from pytorchvideo_b200.engine.lower import lower_only
    from oracle.audio_ref import audio_forward
    out = {}
    for case in TS.AUDIO_CASES:
        mine, x = TS.build_audio_case(case, mine_builders, seed=SEED)
        ref, _ = TS.build_audio_case(case, _RefBuilders, seed=SEED)
        assert list(ref.state_dict().keys()) == list(mine.state_dict().keys()), case
        assert repr(ref) == repr(mine), case
        ref.load_state_dict(mine.state_dict(), strict=True)
        with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
            y = ref([t.clone() for t in x] if isinstance(x, list) else x.clone())
        assert torch.equal(audio_forward(ref, x), y), "oracle != reference on reference modules (%s)" % case
        assert torch.equal(audio_forward(mine, x), y), "oracle != reference on product tree (%s)" % case
        plan, _ = lower_only(ref, x)
        out[case] = {"seed": SEED, "output": y.clone(), "state_checksum": TS.state_checksum(mine),
                     "input_checksum": [TS.tensor_checksum(t) for t in (x if isinstance(x, list) else [x])],
                     "repr": repr(ref), "keys": list(ref.state_dict().keys()),
                     "launches": [(md["name"], md["kind"]) for md in plan.meta]}
        print("%-20s ok  out %s  |out|max %.4f  launches %d" % (case, tuple(y.shape), float(y.abs().max()),
                                                               len(plan.meta)), flush=True)
    torch.save(out, GOLD)


if __name__ == "__main__":
    main()
