"""ORACLE (test infrastructure only): the mobile efficient blocks restated on the CPU.

``EfficientOracle`` is the structural interpreter of oracle/interp.py with handlers for the efficient blocks of the
reference (layers/accelerator/mobile_cpu/, models/accelerator/mobile_cpu/) in their original form, so Efficient X3D
evaluates in the same fp32 CPU arithmetic as every other oracle case.  oracle/gen_golden_efficient.py pins it bit for
bit to the reference's forward, on the reference's module tree and on this package's.
"""
import torch
import torch.nn.functional as F

from oracle.interp import Oracle, _leaf


class EfficientOracle(Oracle):
    def _kernel(self, m, x):                       # convolutions.py: kernel = Sequential(conv, [bn], act)
        return self.run(m.kernel, x)

    f_Conv3dPwBnAct = f_Conv3d3x3x3DwBnAct = f_Conv3dTemporalKernel1BnAct = _kernel
    f_Conv3d3x1x1BnAct = f_Conv3d5x1x1BnAct = _kernel

    def _act(self, m, x):
        # activation_functions.py wraps the activation as .act; the torch / pytorchvideo leaves share the class names
        if hasattr(m, "act"):
            return self.run(m.act, x)
        return F.hardswish(x) if type(m).__name__ == "Hardswish" else _leaf(m, x)

    f_ReLU = f_Swish = f_Identity = f_HardSwish = f_Hardswish = _act

    def f_SqueezeExcitation(self, m, x):           # attention.py: the mobile wrapper holds the fvcore SE as .se
        if hasattr(m, "se"):
            return self.run(m.se, x)
        return super().f_SqueezeExcitation(m, x)

    def f_AdaptiveAvgPool3dOutSize1(self, m, x):   # pool.py
        return self.run(m.pool, x)

    def _model(self, m, x):                        # no_op_convert_block.py; torch's AdaptiveAvgPool3d shares the name
        return self.run(m.model, x) if hasattr(m, "model") else _leaf(m, x)

    f_NoOpConvertBlock = f_FullyConnected = f_AdaptiveAvgPool3d = _model

    def f_X3dBottleneckBlock(self, m, x):          # residual_blocks.py forward
        out = self.run(m.layers, x)
        if m._use_residual:
            if m._res_proj is not None:
                x = self.run(m._res_proj, x)
            out = torch.add(x, out)
        return self.run(m.final_act, out)

    def f_EfficientX3d(self, m, x):                # efficient_x3d.py forward, eval mode
        for s in (m.s1, m.s2, m.s3, m.s4, m.s5):
            x = self.run(s, x)
        if m.enable_head:
            x = self.run(m.head, x)
            x = x.permute((0, 2, 3, 4, 1))
            x = self.run(m.projection, x)
            x = self.run(m.act, x)
            x = x.mean([1, 2, 3])
            x = x.view(x.shape[0], -1)
        return x


def efficient_forward(model, x):
    """Eval-mode fp32 CPU forward of an efficient-block model or block on ``x``."""
    with torch.no_grad():
        return EfficientOracle().run(model, x.detach().float().cpu())
