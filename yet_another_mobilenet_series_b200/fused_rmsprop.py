"""Fused flat-arena RMSprop for sm_90a with the surface of the reference's `utils/rmsprop.py`.

Drop-in contract (SURVEY.md §8b): `torch.optim.Optimizer` subclass, constructor
`(params, lr=1e-2, alpha=0.99, eps=1e-8, eps_inside_sqrt=False, weight_decay=0, momentum=0,
centered=False)` (reference utils/rmsprop.py:31-39), `ValueError` on negative values (:40-50),
`param_groups[0]['lr']` honoured every step (LambdaLR mutates it, reference train.py:103),
per-parameter state `{'step','square_avg','momentum_buffer'[, 'grad_avg']}` (:89-95) that
round-trips through `state_dict()` / `load_state_dict()`.

What is different underneath: every parameter, gradient and state tensor is a VIEW into one flat
fp32 arena (flat_arena.FlatArenaOptimizer, shared with fused_sgd.SGD), so
  * `step()` is ONE kernel (`yamb_rmsprop_step`) instead of ~7 launches x 158 tensors,
  * the gradient all-reduce (reference utils/distributed.py:131-139) runs in place on the flat
    gradient arena with no flatten/unflatten copies and its 1/world is folded into the step,
  * the L2 penalty of `cal_l2_loss('mnas' or 'slimmable')` (utils/optim.py:161-200) and the EMA
    of the weights (utils/optim.py:53-64, train.py:109-114) can be folded into the same pass
    (`fold_l2`, `attach_ema`),
  * a bf16 mirror of the weights is refreshed in the same pass and used directly as the
    tensor-core operand of the block kernels.

Plugin hook: `get_optimizer(model)` is what the reference calls through
`importlib.import_module(FLAGS.optimizer).get_optimizer(model)` (utils/optim.py:277-279).
"""
import ctypes as C

from . import native as nat
from .flat_arena import FlatArenaOptimizer, l2_mask, mnas_l2_mask  # noqa: F401 (public names)


class RMSprop(FlatArenaOptimizer):
    """TF-style RMSprop (eps inside/outside the sqrt, momentum, centered) as one fused kernel."""

    _name = "fused RMSprop"
    _hyper_keys = ("alpha", "eps", "eps_inside_sqrt", "momentum", "centered", "weight_decay")

    def __init__(self, params, lr=1e-2, alpha=0.99, eps=1e-8, eps_inside_sqrt=False,
                 weight_decay=0, momentum=0, centered=False):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: {}".format(lr))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {}".format(eps))
        if not 0.0 <= momentum:
            raise ValueError("Invalid momentum value: {}".format(momentum))
        if not 0.0 <= weight_decay:
            raise ValueError("Invalid weight_decay value: {}".format(weight_decay))
        if not 0.0 <= alpha:
            raise ValueError("Invalid alpha value: {}".format(alpha))
        defaults = dict(lr=lr, momentum=momentum, alpha=alpha, eps=eps,
                        eps_inside_sqrt=eps_inside_sqrt, centered=centered,
                        weight_decay=weight_decay)
        super().__init__(params, defaults)

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("momentum", 0)
            group.setdefault("centered", False)

    # ---- state arenas --------------------------------------------------------------------------
    def _alloc_state(self, A, hp, z):
        A["sq"] = z()
        A["mom"] = z() if hp["momentum"] > 0 else None
        A["gavg"] = z() if hp["centered"] else None

    def _link_state(self, A, p, old, o):
        n = p.numel()
        st = dict(old)
        st["step"] = old.get("step", 0)
        for key, arena in (("square_avg", "sq"), ("momentum_buffer", "mom"), ("grad_avg", "gavg")):
            if A[arena] is None:
                continue
            st[key] = A[arena][o:o + n].view(p.shape)
            if key in old:
                st[key].copy_(old[key])
        return st

    # ---- the step ------------------------------------------------------------------------------
    def _launch(self, A, mask, num_updates, use_device_hyper):
        """One fused update of every parameter (reference utils/rmsprop.py:67-129)."""
        g0 = self.param_groups[0]
        a = nat.Rmsprop()
        a.n = A["n"]
        a.p, a.g, a.sq = A["p"].data_ptr(), A["g"].data_ptr(), A["sq"].data_ptr()
        a.mom = nat.ptr(A["mom"])
        a.grad_avg = nat.ptr(A["gavg"])
        a.ema = nat.ptr(A["ema"])
        a.p_bf16 = A["bf16"].data_ptr()
        a.wd_mask = nat.ptr(mask)
        a.lr, a.alpha, a.eps = g0["lr"], g0["alpha"], g0["eps"]
        a.momentum, a.weight_decay = g0["momentum"], g0["weight_decay"]
        a.l2 = self._l2
        a.grad_scale = self.grad_scale
        a.eps_inside_sqrt = 1 if g0["eps_inside_sqrt"] else 0
        a.centered = 1 if g0["centered"] else 0
        a.ema_m = self.ema_momentum(num_updates) if self._ema_decay is not None else 0.0
        if use_device_hyper:
            a.hyper = self._hyper.data_ptr()
        nat.check(nat.lib().yamb_rmsprop_step(C.byref(a), nat.stream_handle()))

    def _after_step(self, A, inactive):
        for i, p in enumerate(A["plist"]):
            if inactive is None or i not in inactive:
                self.state[p]["step"] += 1


def get_optimizer(model):
    """Plugin entry of the reference (`optimizer: yet_another_mobilenet_series_b200.fused_rmsprop`
    in the yml; utils/optim.py:277-279).  Reads the same FLAGS fields as the reference's own
    rmsprop branch (utils/optim.py:269-275)."""
    from utils.config import FLAGS  # the reference's config singleton, present in its process
    return RMSprop(model.parameters(), lr=FLAGS.lr, alpha=FLAGS.alpha, momentum=FLAGS.momentum,
                   eps=FLAGS.epsilon, eps_inside_sqrt=FLAGS.eps_inside_sqrt, weight_decay=0)
