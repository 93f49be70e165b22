"""BYOL (reference models/byol.py, https://arxiv.org/pdf/2006.07733.pdf) on the engine.

forward(x1, x2) runs, in the reference's order (byol.py:124-143):
  1. the online plan predictor(backbone(x)) for both views, each normalised by pv_rows_l2_normalize;
  2. the momentum update of ``backbone_mmt`` (pv_ema_update, one launch for every parameter) - also in eval mode,
     as the reference, whose update is under no_grad and not gated on ``self.training``;
  3. the momentum plan backbone_mmt(x) for both views, normalised;
  4. pv_contrastive_ce in BYOL mode over the stacked pairs (pred_1, proj_mmt_2) and (pred_2, proj_mmt_1), which is
     (sim_loss(pred_1, proj_mmt_2) + sim_loss(pred_2, proj_mmt_1)) / 2.

The momentum update writes ``backbone_mmt``'s parameters IN PLACE.  The reference rebinds ``param_mmt.data`` to a new
tensor instead; values and state_dict are identical, only ``data_ptr()`` differs.  The momentum plan is compiled once
per input shape as a refreshable plan (engine/refresh.py): after every update pv_weights_refresh re-derives its packed
weights and folded BatchNorm vectors on the device, in the same buffers, and the same CUDA graph is replayed.  A plan
with a constant that is not a pure re-layout of one parameter or a BatchNorm fold is compiled again after every
update instead.  A change of ``backbone_mmt`` from outside (load_state_dict, .to()) compiles the plans again.
"""
import copy
from typing import Callable, Optional

import torch
import torch.nn as nn

from .. import config, contrastive as K
from ..engine import lower as _lower
from ..engine.refresh import WeightsRefresh
from .embedding import EmbeddingChain, check_call


class BYOL(nn.Module):
    def __init__(self, backbone: nn.Module, projector: Optional[nn.Module] = None,
                 predictor: Optional[nn.Module] = None, feature_dim: int = 2048, predictor_inner: int = 4096,
                 mmt: float = 0.99, norm: Callable = nn.SyncBatchNorm) -> None:
        super().__init__()
        self.mmt = mmt
        self.feature_dim = feature_dim
        if projector is not None:
            backbone = nn.Sequential(backbone, projector)
        self.backbone = backbone
        self.backbone_mmt = copy.deepcopy(backbone)
        for p in self.backbone_mmt.parameters():
            p.requires_grad = False
        if predictor is None:
            self.predictor = nn.Sequential(
                nn.Linear(feature_dim, predictor_inner, bias=False),
                norm(predictor_inner),
                nn.ReLU(inplace=True),
                nn.Linear(predictor_inner, feature_dim, bias=True),
            )
        else:
            self.predictor = predictor
        self.__dict__["_pv_state"] = None

    def __getstate__(self):
        """copy.deepcopy / pickle: the compiled plans, their CUDA graphs and refresh tables are derived data."""
        st = dict(self.__dict__)
        st["_pv_state"] = None
        return st

    def update_mmt(self, mmt: float):
        """Set the momentum (momentum annealing)."""
        self.mmt = mmt

    def get_mmt(self) -> float:
        return self.mmt

    def _state(self):
        st = self.__dict__.get("_pv_state")
        params = list(self.backbone.parameters())
        params_mmt = list(self.backbone_mmt.parameters())
        key = tuple((p.data_ptr(), q.data_ptr()) for p, q in zip(params, params_mmt))
        if st is None or st["key"] != key or st["online"].seq[0] is not self.backbone:
            st = self.__dict__["_pv_state"] = {
                "key": key,
                "online": EmbeddingChain(self.backbone, self.predictor),
                "mmt": EmbeddingChain(self.backbone_mmt),
                "ema": None,
                "plans": {},           # momentum plans: key -> (CompiledModel, WeightsRefresh or None)
                "fp": None,
            }
        return st

    def _mmt_plan(self, x):
        """The momentum plan for inputs like ``x`` (compiled once, refreshed in place after every update)."""
        st = self._state()
        ch = st["mmt"]
        fp = ch._pv_fingerprint()
        if st["fp"] != fp:                                 # backbone_mmt changed from outside: compile again
            st["plans"].clear()
            st["fp"] = fp
        key = (tuple(x.shape), x.dtype, x.device.index, config.get_precision(), config.get_use_graph())
        entry = st["plans"].get(key)
        if entry is None:
            cm = _lower.compile_model(ch, x, config.get_precision(), config.get_use_graph())
            entry = st["plans"][key] = (cm, WeightsRefresh.build(cm, ch, x, config.get_precision()))
        return entry[0]

    @torch.no_grad()
    def _momentum_update_backbone(self):
        """backbone_mmt = backbone_mmt * mmt + backbone * (1 - mmt), in place, one launch (pv_ema_update)."""
        st = self._state()
        if st["ema"] is None:
            st["ema"] = K.EmaUpdate([p.data for p in self.backbone_mmt.parameters()],
                                    [p.data for p in self.backbone.parameters()])
        st["ema"](self.mmt)
        for key, (cm, refresh) in list(st["plans"].items()):
            if refresh is None:
                del st["plans"][key]                       # not refreshable: compiled again on its next use
            else:
                refresh()

    def forward_backbone(self, x):
        """F.normalize(predictor(backbone(x)), dim=1) as fp32 rows."""
        check_call(self, x)
        return K.l2_normalize(self._state()["online"].embed(x))

    @torch.no_grad()
    def forward_backbone_mmt(self, x):
        """F.normalize(backbone_mmt(x), dim=1) as fp32 rows."""
        check_call(self, x)
        return K.l2_normalize(self._mmt_embed(x))

    def _mmt_embed(self, x):
        if not torch.is_tensor(x):
            raise RuntimeError("expected a tensor input")
        return self._mmt_plan(x)(x)

    def forward(self, x1: torch.Tensor, x2: torch.Tensor) -> torch.Tensor:
        check_call(self, x1, x2)
        if x1.shape != x2.shape:
            raise RuntimeError("the two views have different shapes %s and %s" % (tuple(x1.shape), tuple(x2.shape)))
        st = self._state()
        B = x1.shape[0]
        pred = st["online"].embed(x1)
        C = pred.shape[1]
        q = torch.empty((2 * B, C), dtype=torch.float32, device=x1.device)
        K.l2_normalize(pred, out=q[:B])
        K.l2_normalize(st["online"].embed(x2), out=q[B:])
        with torch.no_grad():
            self._momentum_update_backbone()
            proj1 = self._mmt_embed(x1)
            k = torch.empty((2 * B, proj1.shape[1]), dtype=torch.float32, device=x1.device)
            K.l2_normalize(proj1, out=k[B:])                # before the second replay overwrites the plan's output
            K.l2_normalize(self._mmt_embed(x2), out=k[:B])
        return K.contrastive_ce(q, k, 1.0, byol=True)
