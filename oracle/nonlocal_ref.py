"""ORACLE (test infrastructure only): the Non-local block restated on the CPU.

``NonLocalOracle`` is the structural interpreter of oracle/interp.py with one more handler, ``f_NonLocal``
(reference layers/nonlocal_net.py:55-94), so whole models that contain Non-local blocks (I3D-NLN: a ResStage whose
res_blocks[i] is Sequential(ResBlock, NonLocal)) evaluate in the same fp32 CPU arithmetic as every other oracle
case.  oracle/gen_golden_nonlocal.py pins it bit for bit to the reference's own module.
"""
import torch
import torch.nn.functional as F

from oracle.interp import Oracle


class NonLocalOracle(Oracle):
    def f_NonLocal(self, m, x):                  # layers/nonlocal_net.py:55-94
        dim_inner = m.conv_theta.out_channels
        N, C, T, H, W = x.size()
        theta = self.run(m.conv_theta, x)
        xp = self.run(m.pool, x)
        phi = self.run(m.conv_phi, xp).view(N, dim_inner, -1)
        g = self.run(m.conv_g, xp).view(N, dim_inner, -1)
        theta_phi = torch.einsum("nct,ncp->ntp", (theta.view(N, dim_inner, -1), phi))
        if m.instantiation == "softmax":
            theta_phi = F.softmax(theta_phi * (dim_inner ** -0.5), dim=2)
        elif m.instantiation == "dot_product":
            theta_phi = theta_phi / theta_phi.shape[2]
        y = torch.einsum("ntg,ncg->nct", (theta_phi, g)).view(N, dim_inner, T, H, W)
        y = self.run(m.conv_out, y)
        if m.norm is not None:
            y = self.run(m.norm, y)
        return x + y


def nonlocal_forward(model, x):
    """Eval-mode fp32 CPU forward of ``model`` (a module tree that may contain Non-local blocks) on the clip ``x``."""
    with torch.no_grad():
        return NonLocalOracle().run(model, x.detach().float().cpu())
