"""Flat-arena machinery shared by the fused optimizers (`fused_rmsprop.RMSprop`, `fused_sgd.SGD`).

Every parameter, gradient and optimizer-state tensor is a VIEW into one flat fp32 arena, so
  * the update is ONE streaming kernel over the arenas instead of several launches per tensor,
  * the gradient all-reduce (reference utils/distributed.py:131-139) runs in place on the flat
    gradient arena and its 1/world is folded into the step (`grad_scale`),
  * the L2 penalty of `cal_l2_loss` (utils/optim.py:161-200) and the EMA of the weights
    (utils/optim.py:53-64, train.py:109-114) are folded into the same pass (`fold_l2`,
    `attach_ema`),
  * a bf16 mirror of the weights is refreshed in the same pass and used directly as the
    tensor-core operand of the block kernels (`_yamb_bf16`), and the kernels accumulate
    parameter gradients straight into the arena (`_yamb_direct`, read by `engine.GradTargets`).

A subclass names its state arenas and per-parameter state (`_alloc_state`, `_link_state`), launches
its kernel (`_launch`) and updates its host-side state after the launch (`_after_step`).
"""
import torch
from torch.optim.optimizer import Optimizer

from . import native as nat

_ALIGN = 8  # elements: keeps every fp32 view 32-byte and every bf16 mirror view 16-byte aligned

# per-element mask bits the optimizer kernels read (include/yamb200.h)
MASK_L2, MASK_NO_GRAD, MASK_FIRST_MOMENTUM = 1, 2, 4


def mnas_l2_mask(named_params):
    """1 where `cal_l2_loss(method='mnas')` regularises (reference utils/optim.py:177-192):
    all 4-D / 2-D weights and the classifier bias; BN gamma/beta are not decayed."""
    mask = {}
    for name, p in named_params:
        if p.dim() in (4, 2):
            mask[name] = True
        else:
            assert p.dim() == 1
            mask[name] = "classifier" in name
    return mask


def slimmable_l2_mask(named_params):
    """1 where `cal_l2_loss(method='slimmable')` regularises (reference utils/optim.py:165-176):
    4-D tensors with shape[1] != 1 and every 2-D tensor.  A rule of shape, not of layer type: the
    depthwise [C,1,k,k] and a one-channel pointwise [Cout,1,1,1] are not decayed, the stem
    [C,3,3,3] is; no 1-D tensor is (classifier bias, BN gamma/beta, SE biases)."""
    return {name: (p.dim() == 4 and p.shape[1] != 1) or p.dim() == 2
            for name, p in named_params}


def l2_mask(named_params, method):
    """{name: decayed?} of `cal_l2_loss(model, wd, method)`; the same errors as the reference for
    the method it leaves unimplemented and for unknown names (utils/optim.py:195-199)."""
    if method == "mnas":
        return mnas_l2_mask(named_params)
    if method == "slimmable":
        return slimmable_l2_mask(named_params)
    if method == "mnas_no_bias":
        raise NotImplementedError("weight_decay method 'mnas_no_bias'")
    raise ValueError("Unknown weight_decay method: {}".format(method))


def ema_momentum(decay, num_updates):
    """EMA momentum of update `num_updates`: min(decay, (1+t)/(10+t)) (reference
    utils/optim.py:56-64); `decay` itself when `num_updates` is None."""
    if num_updates is None:
        return decay
    return min(decay, (1.0 + num_updates) / (10.0 + num_updates))


class FlatArenaOptimizer(Optimizer):
    """`torch.optim.Optimizer` whose parameters, gradients and state live in flat fp32 arenas."""

    _name = "fused optimizer"   # in error messages
    _hyper_keys = ()            # param-group keys (besides lr) that must agree across groups

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._arenas = None
        self._l2 = 0.0
        self._l2_ids = set()
        self._ema_decay = None
        self.grad_scale = 1.0
        self._hyper = None

    # ---- configuration of the folded-in services ---------------------------------------------
    def fold_l2(self, weight_decay, named_params, method="mnas"):
        """Apply d/dp [0.5*wd*sum p^2] = wd*p inside the step for the parameters
        `cal_l2_loss(method)` would regularise ('mnas' or 'slimmable').  Use INSTEAD of adding
        `cal_l2_loss` to the loss."""
        named_params = list(named_params)
        mask = l2_mask(named_params, method)
        self._l2 = float(weight_decay)
        self._l2_ids = {id(p) for n, p in named_params if mask[n]}
        self._arenas = None  # rebuild with the mask

    def attach_ema(self, decay):
        """Maintain shadow = m*shadow + (1-m)*p for every parameter inside the step, with
        m = min(decay, (1+t)/(10+t)) (reference utils/optim.py:56-64).  `ema_shadow(p)` reads it."""
        self._ema_decay = float(decay)
        self._arenas = None

    # ---- subclass hooks ------------------------------------------------------------------------
    def _alloc_state(self, A, hp, z):
        """Allocate the optimizer's state arenas into A (z() -> zeroed fp32 arena)."""
        raise NotImplementedError

    def _link_state(self, A, p, old, o):
        """The per-parameter state dict with its tensors as arena views (offset o); `old` is what
        the state held before (e.g. loaded by load_state_dict).  An empty dict: no entry."""
        raise NotImplementedError

    def _step_marks(self, A, inactive):
        """Extra (parameter index, mask bit) pairs for this step; `inactive`: the indices of the
        parameters without a gradient."""
        return []

    def _launch(self, A, mask, num_updates, use_device_hyper):
        raise NotImplementedError

    def _after_step(self, A, inactive):
        pass

    # ---- flat arenas ---------------------------------------------------------------------------
    def _build(self):
        groups = self.param_groups
        plist = [p for g in groups for p in g["params"]]
        if not plist:
            raise ValueError("optimizer got an empty parameter list")
        dev = plist[0].device
        if dev.type != "cuda":
            raise nat.NativeError("%s runs only on CUDA (no CPU fallback)" % self._name)
        if any(p.dtype != torch.float32 or p.device != dev for p in plist):
            raise nat.NativeError("%s needs fp32 parameters on one device" % self._name)
        hp = {k: groups[0][k] for k in self._hyper_keys}
        for g in groups[1:]:
            if any(g[k] != hp[k] for k in hp) or g["lr"] != groups[0]["lr"]:
                raise nat.NativeError("%s supports one hyper-parameter set" % self._name)
        offs, total = [], 0
        for p in plist:
            offs.append(total)
            total += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        z = lambda dt=torch.float32: torch.zeros(total, device=dev, dtype=dt)
        A = {"p": z(), "g": z(), "n": total, "offs": offs, "plist": plist}
        self._alloc_state(A, hp, z)
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
                st = self._link_state(A, p, dict(self.state.get(p, {})), o)
                if st:
                    self.state[p] = st
                else:
                    self.state.pop(p, None)
                if A["mask"] is not None and id(p) in self._l2_ids:
                    A["mask"][o:o + n] = MASK_L2
            A["bf16"].copy_(A["p"])
            if A["ema"] is not None:
                A["ema"].copy_(A["p"])
        for p in plist:
            p._yamb_bf16_version = p._version     # the mirror is fresh as of this version
        A["gptr"] = [A["g"].data_ptr() + 4 * o for o in offs]
        A["frozen"] = None                        # mask variant used while some step marks apply
        self._hyper = torch.zeros(2, device=dev, dtype=torch.float32)
        self._arenas = A
        return A

    def arenas(self):
        """Flat arenas (built on first use): dict with 'p','g','bf16','ema','n' and the state
        arenas of the subclass."""
        return self._arenas if self._arenas is not None else self._build()

    def ema_shadow(self, p):
        A = self.arenas()
        i = [id(q) for q in A["plist"]].index(id(p))
        o = A["offs"][i]
        return A["ema"][o:o + p.numel()].view(p.shape)

    def load_in_place(self, state_dict, ema=None):
        """`load_state_dict` into the CURRENT arenas: hyper-parameters and per-parameter state are
        copied into the existing views, and `ema` (tensors in parameter order, e.g. the shadows of
        a checkpoint) into the EMA arena.  No arena is rebuilt, so the addresses a captured CUDA
        graph holds stay valid.  State a parameter has no entry for in `state_dict` is zeroed, as
        in a fresh arena."""
        A = self.arenas()
        saved = state_dict["param_groups"]
        if len(saved) != len(self.param_groups) or \
                any(len(g["params"]) != len(s["params"]) for g, s in zip(self.param_groups, saved)):
            raise ValueError("loaded state dict has a different parameter layout than the optimizer")
        index = {id(p): i for g, s in zip(self.param_groups, saved)
                 for p, i in zip(g["params"], s["params"])}
        for g, s in zip(self.param_groups, saved):
            g.update({k: v for k, v in s.items() if k != "params"})
        with torch.no_grad():
            for p, o in zip(A["plist"], A["offs"]):
                old = state_dict["state"].get(index[id(p)], {})
                st = self._link_state(A, p, old, o)
                for k, v in st.items():
                    if torch.is_tensor(v) and k not in old:
                        v.zero_()
                if st:
                    self.state[p] = st
                else:
                    self.state.pop(p, None)
            if ema is not None:
                if A["ema"] is None:
                    raise ValueError("load_in_place: this optimizer keeps no EMA (attach_ema)")
                shadows = list(ema)
                if len(shadows) != len(A["plist"]):
                    raise ValueError("load_in_place: %d EMA shadows for %d parameters"
                                     % (len(shadows), len(A["plist"])))
                for p, o, s in zip(A["plist"], A["offs"], shadows):
                    A["ema"][o:o + p.numel()].view(p.shape).copy_(s)
        self._state_loaded(A)

    def _state_loaded(self, A):
        """Hook: host-side bookkeeping derived from `self.state` is stale (load_in_place)."""
        A["frozen"] = None

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
        the step exactly like the reference does (utils/rmsprop.py:77-78, torch.optim.SGD).
        Returns the per-element mask to hand to the kernel and the set of skipped indices (None
        when the plain mask applies)."""
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
        marks = [(i, MASK_NO_GRAD) for i in inactive] + self._step_marks(A, set(inactive))
        if not marks:
            return A["mask"], None
        key = tuple(marks)
        if A["frozen"] is None or A["frozen"][0] != key:
            m = A["mask"].clone() if A["mask"] is not None else \
                torch.zeros(A["n"], device=A["p"].device, dtype=torch.uint8)
            for i, bit in marks:
                o = A["offs"][i]
                m[o:o + A["plist"][i].numel()] |= bit
            A["frozen"] = (key, m)
        return A["frozen"][1], set(inactive)

    def load_state_dict(self, state_dict):
        """torch's load_state_dict, then the loaded state is linked into fresh arenas.  The EMA of
        the weights is not part of an optimizer state_dict: the shadows are carried over (use
        `load_in_place` to load them too and keep the arenas)."""
        old = self._arenas
        super().load_state_dict(state_dict)
        self._arenas = None  # re-link loaded state tensors into fresh arenas on next use
        A = self.arenas()
        if old is not None and old["ema"] is not None and A["ema"] is not None:
            A["ema"].copy_(old["ema"])

    # ---- the step ------------------------------------------------------------------------------
    def set_hyper_device(self, lr, ema_m):
        """Write lr / EMA momentum to the device scalars read by a CUDA-graph-captured step."""
        self._hyper.copy_(torch.tensor([lr, ema_m], dtype=torch.float32), non_blocking=True)

    def ema_momentum(self, num_updates):
        return ema_momentum(self._ema_decay, num_updates)

    @torch.no_grad()
    def step(self, closure=None, num_updates=None, use_device_hyper=False):
        """One fused update of every parameter.

        `num_updates`: global step used by the EMA warm-up rule (train.py:109-114 passes
        FLAGS._global_step AFTER incrementing it)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        A = self.arenas()
        mask, inactive = self._collect_grads(A)
        self._launch(A, mask, num_updates, use_device_hyper)
        self._after_step(A, inactive)
        return loss
