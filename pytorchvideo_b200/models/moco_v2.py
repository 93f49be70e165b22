"""MoCo v2 (reference pytorchvideo_trainer module/moco_v2.py, https://arxiv.org/abs/1911.05722) on the engine.

``MOCO`` keeps the reference's module tree and state_dict keys (``backbone`` and ``backbone_mmt``, each an
nn.Sequential of trunk and projector).  ``forward`` is the online plan followed by pv_rows_l2_normalize.
``forward_backbone_mmt`` replays a refreshable momentum plan, as BYOL's (engine/refresh.py): after every
``momentum_update_backbone`` (pv_ema_update, one launch for every parameter, paired by name as the reference's dict
pairs them) pv_weights_refresh rewrites the plan's constants in place and the same CUDA graph is replayed.  The
reference computes ``src * (1 - m) + dst * m``; the kernel's ``dst * m + src * (1 - m)`` is the same bits, because IEEE
addition commutes.  The update writes ``backbone_mmt`` IN PLACE where the reference rebinds ``.data``.

``MoCoQueue`` is the state and objective of the trainer's ``MOCOV2Module``: its ``queue_x`` and ``ptr`` buffers, the
keys, the per-view losses of ``training_step`` (pv_queue_ce: one streamed pass over the queue per view, the logits
never stored) and the enqueue.  Eval mode only, in one process: training mode raises RuntimeError and an initialised
``torch.distributed`` with more than one rank raises NotImplementedError (shuffle-BN across ranks is not implemented).
"""
import math
from typing import Callable, List, Optional, Tuple

import torch
import torch.nn as nn

from .. import config, contrastive as K
from ..engine import lower as _lower
from ..engine.refresh import WeightsRefresh
from ..losses.contrastive_loss import ContrastiveLoss
from .embedding import EmbeddingChain, check_call
from .resnet import create_resnet
from .weight_init import init_net_weights


def _single_process():
    if torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
        raise NotImplementedError("MoCo on the engine runs in one process: shuffle-BN across ranks is not implemented")


def create_mlp_util(dim_in: int, dim_out: int, mlp_dim: int, num_layers: int, norm: Callable, bias: bool = True,
                    xavier_init: bool = True) -> nn.Module:
    """Linear -> [norm] -> ReLU ... -> Linear (ssl_helper.py:21-64); each Linear but a lone one carries the
    ``xavier_init`` attribute that init_net_weights reads."""
    if num_layers == 1:
        return nn.Linear(dim_in, dim_out)
    b = False if norm is not None else bias
    mlp_layers = [nn.Linear(dim_in, mlp_dim, bias=b)]
    mlp_layers[-1].xavier_init = xavier_init
    for i in range(1, num_layers):
        if norm:
            mlp_layers.append(norm(mlp_dim))
        mlp_layers.append(nn.ReLU(inplace=True))
        if i == num_layers - 1:
            d = dim_out
            b = bias
        else:
            d = mlp_dim
        mlp_layers.append(nn.Linear(mlp_dim, d, bias=b))
        mlp_layers[-1].xavier_init = xavier_init
    return nn.Sequential(*mlp_layers)


def create_moco_resnet_50(backbone_creator: Callable = create_resnet, backbone_embed_dim: int = 128,
                          head_pool: Callable = nn.AdaptiveAvgPool3d, head_output_size: Tuple[int, int, int] = (1, 1, 1),
                          head_activation: Callable = None, dropout_rate: float = 0.0, projector_dim_in: int = 2048,
                          projector_inner_dim: int = 2048, projector_depth: int = 3,
                          projector_norm: Optional[Callable] = None, mmt: float = 0.994) -> nn.Module:
    def _make_backbone_and_projector():
        backbone = backbone_creator(dropout_rate=dropout_rate, head_activation=head_activation,
                                    head_output_with_global_average=True, head_pool=head_pool,
                                    head_output_size=head_output_size, stem_conv_kernel_size=(1, 7, 7),
                                    head_pool_kernel_size=(8, 7, 7))
        backbone.blocks[-1].proj = None
        projector = create_mlp_util(projector_dim_in, backbone_embed_dim, projector_inner_dim, projector_depth,
                                    norm=projector_norm)
        return backbone, projector

    backbone, projector = _make_backbone_and_projector()
    backbone_mmt, projector_mmt = _make_backbone_and_projector()
    return MOCO(mmt=mmt, backbone=backbone, projector=projector, backbone_mmt=backbone_mmt,
                projector_mmt=projector_mmt)


class MOCO(nn.Module):
    def __init__(self, mmt: float, backbone: nn.Module, backbone_mmt: nn.Module, projector: Optional[nn.Module] = None,
                 projector_mmt: Optional[nn.Module] = None) -> None:
        super().__init__()
        self.mmt: float = mmt
        if projector is not None:
            backbone = nn.Sequential(backbone, projector)
        init_net_weights(backbone)
        self.backbone = backbone
        if projector_mmt is not None:
            backbone_mmt = nn.Sequential(backbone_mmt, projector_mmt)
        init_net_weights(backbone_mmt)
        self.backbone_mmt = backbone_mmt
        for p in self.backbone_mmt.parameters():
            p.requires_grad = False
        self._copy_weights_to_backbone_mmt()
        self.__dict__["_pv_state"] = None

    def __getstate__(self):
        """copy.deepcopy / pickle: the compiled plans, their CUDA graphs and refresh tables are derived data."""
        st = dict(self.__dict__)
        st["_pv_state"] = None
        return st

    def _copy_weights_to_backbone_mmt(self) -> None:
        dist = dict(self.backbone.named_parameters())
        with torch.no_grad():
            for name, p in self.backbone_mmt.named_parameters():
                p.data.copy_(dist[name].data)

    def _pairs(self):
        dist = dict(self.backbone.named_parameters())
        mm = list(self.backbone_mmt.named_parameters())
        return [p for _, p in mm], [dist[name] for name, _ in mm]

    def _state(self):
        st = self.__dict__.get("_pv_state")
        dst, src = self._pairs()
        key = tuple((p.data_ptr(), q.data_ptr()) for p, q in zip(dst, src))
        if st is None or st["key"] != key or st["online"].seq[0] is not self.backbone:
            st = self.__dict__["_pv_state"] = {
                "key": key,
                "online": EmbeddingChain(self.backbone),
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
    def momentum_update_backbone(self) -> None:
        """backbone_mmt = backbone * (1 - mmt) + backbone_mmt * mmt, in place, one launch, then the momentum plans are
        refreshed (or, when not refreshable, dropped and compiled again on their next use)."""
        st = self._state()
        if st["ema"] is None:
            dst, src = self._pairs()
            st["ema"] = K.EmaUpdate([p.data for p in dst], [p.data for p in src])
        st["ema"](self.mmt)
        for key, (cm, refresh) in list(st["plans"].items()):
            if refresh is None:
                del st["plans"][key]
            else:
                refresh()

    def mmt_embed(self, x):
        """backbone_mmt(x) as fp32 rows, from the momentum plan's output buffer (valid until its next replay)."""
        check_call(self, x)
        return self._mmt_plan(x)(x)

    @torch.no_grad()
    def forward_backbone_mmt(self, x: torch.Tensor) -> torch.Tensor:
        """F.normalize(backbone_mmt(x), dim=1) as fp32 rows."""
        return K.l2_normalize(self.mmt_embed(x))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """F.normalize(backbone(x), dim=1) as fp32 rows."""
        check_call(self, x)
        return K.l2_normalize(self._state()["online"].embed(x))


class MoCoQueue(nn.Module):
    """The key queue of MOCOV2Module (moco_v2.py:245-257, 291-427): buffers ``ptr`` and ``queue_x`` (k, dim), drawn as
    the reference draws them (torch.rand on the CPU generator)."""

    def __init__(self, dim: int, k: int, batch_shuffle: bool = True, local_shuffle_bn: bool = False) -> None:
        super().__init__()
        self.dim = dim
        self.k = k
        self.batch_shuffle_on = batch_shuffle
        self.local_shuffle_bn = local_shuffle_bn
        self.register_buffer("ptr", torch.tensor([0]))
        stdv = 1.0 / math.sqrt(self.dim / 3)
        self.register_buffer("queue_x", torch.rand(self.k, self.dim).mul_(2 * stdv).add_(-stdv))

    @torch.no_grad()
    def compute_keys(self, model: MOCO, inputs: List[torch.Tensor]) -> torch.Tensor:
        """The momentum keys of every view as one fp32 (V, B, dim) tensor.  Under batch_shuffle the reference's
        torch.randperm is drawn once per view, so the RNG stream stays the reference's; the permutation itself is not
        applied: in eval mode BatchNorm uses running statistics, so each key depends only on its own clip and
        permute -> momentum backbone -> unpermute gives the same keys."""
        _single_process()
        keys = None
        for v, sub_x in enumerate(inputs):
            if self.batch_shuffle_on:
                torch.randperm(sub_x.shape[0])
            emb = model.mmt_embed(sub_x)
            if keys is None:
                keys = torch.empty((len(inputs),) + tuple(emb.shape), dtype=torch.float32, device=emb.device)
            K.l2_normalize(emb, out=keys[v])
        return keys

    @torch.no_grad()
    def dequeue_and_enqueue(self, keys) -> None:
        """Write each view's keys at ``ptr`` in order, wrapping at k (moco_v2.py:407-427)."""
        assert len(keys) > 0, "need to have multiple views for adding them to queue"
        ptr = int(self.ptr.item())
        for key in keys:
            num_items = int(key.size(0))
            assert self.k % num_items == 0, "Queue size should be a multiple of batchsize"
            assert ptr + num_items <= self.k
            self.queue_x[ptr:ptr + num_items, :].copy_(key)
            ptr += num_items
            if ptr == self.k:
                ptr = 0
            self.ptr[0] = ptr

    @torch.no_grad()
    def step(self, model: MOCO, inputs: List[torch.Tensor], loss: ContrastiveLoss, knn_memory=None,
             video_index: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
        """The sequence of MOCOV2Module.training_step (moco_v2.py:304-333) without the optimizer: the momentum update,
        the keys, one loss per view (the queue as it was before the step), the kNN memory update with the last view's
        embedding, and the enqueue.  Returns the per-view losses the reference hands to manual_backward."""
        _single_process()
        if not isinstance(loss, ContrastiveLoss):
            raise NotImplementedError("MoCoQueue.step computes ContrastiveLoss; got %s" % type(loss).__name__)
        if self.queue_x.device.type != "cuda":
            raise RuntimeError("the MoCo queue is on the CPU: move it with .to()")
        model.momentum_update_backbone()
        keys = self.compute_keys(model, inputs)
        assert len(inputs) > 1, "Length of keys cannot be zero"
        losses = []
        proj = None
        for v, vids in enumerate(inputs):
            proj = model(vids)
            losses.append(K.queue_ce(proj, self.queue_x, keys, loss.temperature, skip_view=v, reduction=loss.reduction))
        if knn_memory is not None:
            knn_memory.update(proj, video_index)
        self.dequeue_and_enqueue(keys)
        return losses
