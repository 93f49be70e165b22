"""ORACLE (test infrastructure only): the audio blocks restated on the CPU.

``AudioOracle`` is the structural interpreter of oracle/interp.py with two more handlers, ``f_SeparableBottleneckBlock``
(reference models/resnet.py:1257-1285) and ``f_FuseAudioToFastSlow`` (models/audio_visual_slowfast.py:406-418, without
the debug print); the acoustic stem's ConvReduce3D(sum) runs through the inherited ``f_ConvReduce3D``.  So AVSlowFast
and the acoustic ResNet evaluate in the same fp32 CPU arithmetic as every other oracle case.  oracle/gen_golden_audio.py
pins it bit for bit to the reference's forward, on the reference's module tree and on this package's.
"""
import torch

from oracle.interp import Oracle


class AudioOracle(Oracle):
    def f_SeparableBottleneckBlock(self, m, x):  # models/resnet.py:1257-1285
        x = self.run(m.act_a, self.run(m.norm_a, self.run(m.conv_a, x)))
        outs = [self.run(a, self.run(n, self.run(c, x))) for c, n, a in zip(m.conv_b, m.norm_b, m.act_b)]
        if m.reduce_method == "sum":
            x = torch.stack(outs, dim=0).sum(dim=0, keepdim=False)
        else:
            x = torch.cat(outs, dim=1)
        return self.run(m.norm_c, self.run(m.conv_c, x))

    def f_FuseAudioToFastSlow(self, m, x):       # models/audio_visual_slowfast.py:406-418
        x_s, x_f, x_a = x[0], x[1], x[2]
        fuse = self.run(m.block_fast_to_slow, x_f)
        fuse_a = self.run(m.block_audio_to_fastslow, torch.mean(x_a, dim=-1, keepdim=True))
        return [fuse_a + torch.cat([x_s, fuse], 1), x_f, x_a]


def audio_forward(model, x):
    """Eval-mode fp32 CPU forward of ``model`` (an audio model or block) on ``x`` (a tensor or a list of pathways)."""
    with torch.no_grad():
        if isinstance(x, (list, tuple)):
            x = [t.detach().float().cpu() for t in x]
        else:
            x = x.detach().float().cpu()
        return AudioOracle().run(model, x)
