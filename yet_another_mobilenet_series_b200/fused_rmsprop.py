"""Fused flat-arena RMSprop for sm_90a with the surface of the reference's `utils/rmsprop.py`.

Drop-in contract (SURVEY.md §8b): `torch.optim.Optimizer` subclass, constructor
`(params, lr=1e-2, alpha=0.99, eps=1e-8, eps_inside_sqrt=False, weight_decay=0, momentum=0,
centered=False)` (reference utils/rmsprop.py:31-39), `ValueError` on negative values (:40-50),
`param_groups[0]['lr']` honoured every step (LambdaLR mutates it, reference train.py:103),
per-parameter state `{'step','square_avg','momentum_buffer'[, 'grad_avg']}` (:89-95) that
round-trips through `state_dict()` / `load_state_dict()`.

What is different underneath: every parameter, gradient and state tensor is a VIEW into one flat
fp32 arena, so
  * `step()` is ONE kernel (`yamb_rmsprop_step`) instead of ~7 launches x 158 tensors,
  * the gradient all-reduce (reference utils/distributed.py:131-139) runs in place on the flat
    gradient arena with no flatten/unflatten copies and its 1/world is folded into the step,
  * the L2 penalty of `cal_l2_loss('mnas')` (utils/optim.py:177-200) and the EMA of the weights
    (utils/optim.py:53-64, train.py:109-114) can be folded into the same pass (`fold_l2`,
    `attach_ema`),
  * a bf16 mirror of the weights is refreshed in the same pass and used directly as the
    tensor-core operand of the block kernels.

Plugin hook: `get_optimizer(model)` is what the reference calls through
`importlib.import_module(FLAGS.optimizer).get_optimizer(model)` (utils/optim.py:277-279).
"""
import ctypes as C

import torch
from torch.optim.optimizer import Optimizer

from . import native as nat

_ALIGN = 8  # elements: keeps every fp32 view 32-byte and every bf16 mirror view 16-byte aligned


def mnas_l2_mask(named_params):
    """1 where `cal_l2_loss(method='mnas')` regularises (reference utils/optim.py:180-191):
    all 4-D / 2-D weights and the classifier bias; BN gamma/beta are not decayed."""
    mask = {}
    n_cls_bias = 0
    for name, p in named_params:
        if p.dim() in (4, 2):
            mask[name] = True
        else:
            assert p.dim() == 1
            is_cls = "classifier" in name
            n_cls_bias += int(is_cls)
            mask[name] = is_cls
    return mask


class RMSprop(Optimizer):
    """TF-style RMSprop (eps inside/outside the sqrt, momentum, centered) as one fused kernel."""

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
        self._arenas = None
        self._l2 = 0.0
        self._l2_ids = set()
        self._ema_decay = None
        self._ema_step_fn = None
        self.grad_scale = 1.0
        self._hyper = None

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("momentum", 0)
            group.setdefault("centered", False)

    # ---- configuration of the folded-in services ---------------------------------------------
    def fold_l2(self, weight_decay, named_params, method="mnas"):
        """Apply d/dp [0.5*wd*sum p^2] = wd*p inside the step for the parameters
        `cal_l2_loss(method)` would regularise.  Use INSTEAD of adding `cal_l2_loss` to the loss."""
        if method != "mnas":
            raise ValueError("Unknown weight_decay method: {}".format(method))
        named_params = list(named_params)
        mask = mnas_l2_mask(named_params)
        self._l2 = float(weight_decay)
        self._l2_ids = {id(p) for n, p in named_params if mask[n]}
        self._arenas = None  # rebuild with the mask

    def attach_ema(self, decay):
        """Maintain shadow = m*shadow + (1-m)*p for every parameter inside the step, with
        m = min(decay, (1+t)/(10+t)) (reference utils/optim.py:56-64).  `ema_shadow(p)` reads it."""
        self._ema_decay = float(decay)
        self._arenas = None

    # ---- flat arenas ---------------------------------------------------------------------------
    def _build(self):
        groups = self.param_groups
        plist = [p for g in groups for p in g["params"]]
        if not plist:
            raise ValueError("optimizer got an empty parameter list")
        dev = plist[0].device
        if dev.type != "cuda":
            raise nat.NativeError("fused RMSprop runs only on CUDA (no CPU fallback)")
        if any(p.dtype != torch.float32 or p.device != dev for p in plist):
            raise nat.NativeError("fused RMSprop needs fp32 parameters on one device")
        hp = {k: groups[0][k] for k in ("alpha", "eps", "eps_inside_sqrt", "momentum",
                                        "centered", "weight_decay")}
        for g in groups[1:]:
            if any(g[k] != hp[k] for k in hp) or g["lr"] != groups[0]["lr"]:
                raise nat.NativeError("fused RMSprop supports one hyper-parameter set")
        offs, total = [], 0
        for p in plist:
            offs.append(total)
            total += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        z = lambda dt=torch.float32: torch.zeros(total, device=dev, dtype=dt)
        A = {"p": z(), "g": z(), "sq": z(), "n": total, "offs": offs, "plist": plist}
        A["mom"] = z() if hp["momentum"] > 0 else None
        A["gavg"] = z() if hp["centered"] else None
        A["bf16"] = z(torch.bfloat16)
        A["ema"] = z() if self._ema_decay is not None else None
        A["mask"] = None
        if self._l2 > 0:
            A["mask"] = torch.zeros(total, device=dev, dtype=torch.uint8)
        with torch.no_grad():
            for p, o in zip(plist, offs):
                n = p.numel()
                view = A["p"][o:o + n].view(p.shape)
                view.copy_(p.data)
                p.data = view
                gview = A["g"][o:o + n].view(p.shape)
                if p.grad is not None:
                    gview.copy_(p.grad)
                p.grad = gview
                p._yamb_direct = True
                p._yamb_bf16 = A["bf16"][o:o + n].view(p.shape)
                st = self.state[p]
                old = dict(st)
                st["step"] = old.get("step", 0)
                st["square_avg"] = A["sq"][o:o + n].view(p.shape)
                if "square_avg" in old:
                    st["square_avg"].copy_(old["square_avg"])
                if A["mom"] is not None:
                    st["momentum_buffer"] = A["mom"][o:o + n].view(p.shape)
                    if "momentum_buffer" in old:
                        st["momentum_buffer"].copy_(old["momentum_buffer"])
                if A["gavg"] is not None:
                    st["grad_avg"] = A["gavg"][o:o + n].view(p.shape)
                    if "grad_avg" in old:
                        st["grad_avg"].copy_(old["grad_avg"])
                if A["mask"] is not None and id(p) in self._l2_ids:
                    A["mask"][o:o + n] = 1
            A["bf16"].copy_(A["p"])
            if A["ema"] is not None:
                A["ema"].copy_(A["p"])
        for p in plist:
            p._yamb_bf16_version = p._version     # the mirror is fresh as of this version
        A["gptr"] = [A["g"].data_ptr() + 4 * o for o in offs]
        A["frozen"] = None                        # mask variant used while some p.grad is None
        self._hyper = torch.zeros(2, device=dev, dtype=torch.float32)
        self._arenas = A
        return A

    def arenas(self):
        """Flat arenas (built on first use): dict with 'p','g','sq','mom','bf16','ema','n'."""
        return self._arenas if self._arenas is not None else self._build()

    def ema_shadow(self, p):
        A = self.arenas()
        i = [id(q) for q in A["plist"]].index(id(p))
        o = A["offs"][i]
        return A["ema"][o:o + p.numel()].view(p.shape)

    def zero_grad(self, set_to_none=True):
        """Zero the flat gradient arena; the `.grad` views are kept (setting them to None would
        detach the parameters from the arena the kernels accumulate into)."""
        A = self.arenas()
        A["g"].zero_()
        # re-attach views dropped by someone else's zero_grad(set_to_none=True)
        for p, o in zip(A["plist"], A["offs"]):
            if p.grad is None:
                p.grad = A["g"][o:o + p.numel()].view(p.shape)

    def sync_mirror(self):
        """Re-cast the bf16 mirror of every parameter whose fp32 master was written in place by
        anybody but `step()` (load_state_dict, broadcast, re-init: they bump `_version`).  Cheap
        host loop; TrainStep calls it before every (graph-replayed) iteration."""
        A = self.arenas()
        stale = [p for p in A["plist"] if p._yamb_bf16_version != p._version]
        with torch.no_grad():
            for p in stale:
                p._yamb_bf16.copy_(p)
                p._yamb_bf16_version = p._version
        return len(stale)

    def _collect_grads(self, A):
        """Make the flat gradient arena reflect every `p.grad` (ADVICE r1): a `.grad` that is no
        longer the arena view (model.zero_grad(set_to_none=True) followed by autograd allocating a
        fresh tensor) is copied in and re-attached; a parameter whose grad is None is skipped by
        the step exactly like the reference does (utils/rmsprop.py:77-78).  Returns the per-element
        mask to hand to the kernel."""
        inactive = []
        for i, p in enumerate(A["plist"]):
            g = p.grad
            if g is None or not p.requires_grad:
                inactive.append(i)
            elif g.data_ptr() != A["gptr"][i]:
                o = A["offs"][i]
                view = A["g"][o:o + p.numel()].view(p.shape)
                view.copy_(g)
                p.grad = view
        if not inactive:
            return A["mask"], None
        key = tuple(inactive)
        if A["frozen"] is None or A["frozen"][0] != key:
            m = A["mask"].clone() if A["mask"] is not None else \
                torch.zeros(A["n"], device=A["p"].device, dtype=torch.uint8)
            for i in inactive:
                o = A["offs"][i]
                m[o:o + A["plist"][i].numel()] |= 2
            A["frozen"] = (key, m)
        return A["frozen"][1], set(inactive)

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._arenas = None  # re-link loaded state tensors into fresh arenas on next use
        self.arenas()

    # ---- the step ------------------------------------------------------------------------------
    def set_hyper_device(self, lr, ema_m):
        """Write lr / EMA momentum to the device scalars read by a CUDA-graph-captured step."""
        self._hyper.copy_(torch.tensor([lr, ema_m], dtype=torch.float32), non_blocking=True)

    def ema_momentum(self, num_updates):
        d = self._ema_decay
        return d if num_updates is None else min(d, (1.0 + num_updates) / (10.0 + num_updates))

    @torch.no_grad()
    def step(self, closure=None, num_updates=None, use_device_hyper=False):
        """One fused update of every parameter (reference utils/rmsprop.py:67-129).

        `num_updates`: global step used by the EMA warm-up rule (train.py:109-114 passes
        FLAGS._global_step AFTER incrementing it)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        A = self.arenas()
        g0 = self.param_groups[0]
        a = nat.Rmsprop()
        a.n = A["n"]
        a.p, a.g, a.sq = A["p"].data_ptr(), A["g"].data_ptr(), A["sq"].data_ptr()
        a.mom = nat.ptr(A["mom"])
        a.grad_avg = nat.ptr(A["gavg"])
        a.ema = nat.ptr(A["ema"])
        a.p_bf16 = A["bf16"].data_ptr()
        mask, inactive = self._collect_grads(A)
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
        for i, p in enumerate(A["plist"]):
            if inactive is None or i not in inactive:
                self.state[p]["step"] += 1
        return loss


def get_optimizer(model):
    """Plugin entry of the reference (`optimizer: yet_another_mobilenet_series_b200.fused_rmsprop`
    in the yml; utils/optim.py:277-279).  Reads the same FLAGS fields as the reference's own
    rmsprop branch (utils/optim.py:269-275)."""
    from utils.config import FLAGS  # the reference's config singleton, present in its process
    return RMSprop(model.parameters(), lr=FLAGS.lr, alpha=FLAGS.alpha, momentum=FLAGS.momentum,
                   eps=FLAGS.epsilon, eps_inside_sqrt=FLAGS.eps_inside_sqrt, weight_decay=0)
