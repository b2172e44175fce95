"""Fused flat-arena SGD for sm_90a with the surface of `torch.optim.SGD`.

The reference's `optimizer: sgd` (utils/optim.py:262-267; apps/mobilenet/default.yml: nesterov,
momentum 0.9, `weight_decay_method: slimmable`) builds `torch.optim.SGD(lr, momentum, nesterov,
weight_decay=0)` and adds `cal_l2_loss` to the loss.  Here:
  * the constructor is torch's `(params, lr=1e-3, momentum=0, dampening=0, weight_decay=0,
    nesterov=False, *, maximize=False, foreach=None, differentiable=False, fused=None)` with the
    same `ValueError`s; `maximize` and `differentiable` are not supported (NativeError), `foreach`
    and `fused` are accepted and ignored;
  * `step()` is ONE kernel (`yamb_sgd_step`) over the flat arenas of flat_arena.py, with the L2
    penalty (`fold_l2`, 'mnas' or 'slimmable'), the 1/world mean (`grad_scale`), the EMA of the
    weights (`attach_ema`) and the bf16 weight mirror folded in;
  * the state is torch's: `{'momentum_buffer': tensor}` for a parameter that has been stepped with
    momentum > 0, nothing otherwise, so `state_dict()`s load into `torch.optim.SGD` and back.

Plugin hook: `optimizer: yet_another_mobilenet_series_b200.fused_sgd` in the yml; the reference
then calls `get_optimizer(model)` (utils/optim.py:277-279).
"""
import ctypes as C

import torch

from . import native as nat
from .flat_arena import MASK_FIRST_MOMENTUM, FlatArenaOptimizer


class SGD(FlatArenaOptimizer):
    """SGD with momentum / dampening / nesterov / weight_decay as one fused kernel."""

    _name = "fused SGD"
    _hyper_keys = ("momentum", "dampening", "weight_decay", "nesterov")

    def __init__(self, params, lr=1e-3, momentum=0, dampening=0, weight_decay=0, nesterov=False,
                 *, maximize=False, foreach=None, differentiable=False, fused=None):
        # torch/optim/sgd.py: the same checks in the same order
        if isinstance(lr, torch.Tensor) and lr.numel() != 1:
            raise ValueError("Tensor lr must be 1-element")
        if lr < 0.0:
            raise ValueError("Invalid learning rate: {}".format(lr))
        if momentum < 0.0:
            raise ValueError("Invalid momentum value: {}".format(momentum))
        if weight_decay < 0.0:
            raise ValueError("Invalid weight_decay value: {}".format(weight_decay))
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        if maximize or differentiable:
            raise nat.NativeError("fused SGD supports neither maximize nor differentiable")
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay,
                        nesterov=nesterov, maximize=maximize, foreach=foreach,
                        differentiable=differentiable, fused=fused)
        super().__init__(params, defaults)

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("nesterov", False)
            group.setdefault("maximize", False)
            group.setdefault("foreach", None)
            group.setdefault("differentiable", False)
            group.setdefault("fused", False)

    # ---- state arenas --------------------------------------------------------------------------
    def _alloc_state(self, A, hp, z):
        A["mom"] = z() if hp["momentum"] > 0 else None
        A["fresh"] = None   # indices of the parameters without a momentum buffer yet

    def _link_state(self, A, p, old, o):
        st = dict(old)
        if A["mom"] is None:
            return st
        buf = st.pop("momentum_buffer", None)
        if buf is not None:           # a buffer exists only once the parameter has been stepped
            st["momentum_buffer"] = A["mom"][o:o + p.numel()].view(p.shape)
            st["momentum_buffer"].copy_(buf)
        return st

    def _step_marks(self, A, inactive):
        if A["mom"] is None:
            return []
        if A["fresh"] is None:
            A["fresh"] = [i for i, p in enumerate(A["plist"])
                          if "momentum_buffer" not in self.state.get(p, {})]
        # torch creates the buffer as a copy of the gradient on the parameter's first step
        return [(i, MASK_FIRST_MOMENTUM) for i in A["fresh"] if i not in inactive]

    # ---- the step ------------------------------------------------------------------------------
    def _launch(self, A, mask, num_updates, use_device_hyper):
        """One fused update of every parameter (torch.optim.SGD.step, _single_tensor_sgd)."""
        g0 = self.param_groups[0]
        if g0["maximize"] or g0["differentiable"]:
            raise nat.NativeError("fused SGD supports neither maximize nor differentiable")
        a = nat.Sgd()
        a.n = A["n"]
        a.p, a.g = A["p"].data_ptr(), A["g"].data_ptr()
        a.mom = nat.ptr(A["mom"])
        a.ema = nat.ptr(A["ema"])
        a.p_bf16 = A["bf16"].data_ptr()
        a.wd_mask = nat.ptr(mask)
        a.lr = float(g0["lr"])
        a.momentum, a.dampening = g0["momentum"], g0["dampening"]
        a.weight_decay = float(g0["weight_decay"])
        a.l2 = self._l2
        a.grad_scale = self.grad_scale
        a.nesterov = 1 if g0["nesterov"] else 0
        a.ema_m = self.ema_momentum(num_updates) if self._ema_decay is not None else 0.0
        if use_device_hyper:
            a.hyper = self._hyper.data_ptr()
        nat.check(nat.lib().yamb_sgd_step(C.byref(a), nat.stream_handle()))

    def _after_step(self, A, inactive):
        if A["mom"] is None or not A["fresh"]:
            return
        left = []
        for i in A["fresh"]:
            if inactive is not None and i in inactive:
                left.append(i)
                continue
            p, o = A["plist"][i], A["offs"][i]
            self.state[p]["momentum_buffer"] = A["mom"][o:o + p.numel()].view(p.shape)
        A["fresh"] = left


def get_optimizer(model):
    """Plugin entry of the reference (`optimizer: yet_another_mobilenet_series_b200.fused_sgd` in
    the yml; utils/optim.py:277-279).  Reads the same FLAGS fields as the reference's own sgd
    branch (utils/optim.py:262-267), with weight_decay=0: the L2 term is `cal_l2_loss` or
    `fold_l2`."""
    from utils.config import FLAGS  # the reference's config singleton, present in its process
    return SGD(model.parameters(), lr=FLAGS.lr, momentum=FLAGS.momentum, nesterov=FLAGS.nesterov,
               weight_decay=0)
