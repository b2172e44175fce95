"""ORACLE of the SGD recipe — test infrastructure only (never imported by the product path).

The reference's `optimizer: sgd` (utils/optim.py:262-267) with `weight_decay_method: slimmable`
(utils/optim.py:161-176), as in apps/mobilenet/default.yml.  Extends the unchanged `oracle`
package:

  sgd_step         numpy float32 restatement of torch.optim.SGD.step (torch/optim/sgd.py,
                   _single_tensor_sgd), line by line
  l2_decay_mask    `oracle.optim.l2_decay_mask` plus the 'slimmable' rule
  l2_loss_slimmable   cal_l2_loss(method='slimmable') on stock torch
  RefTrainer       `oracle.torch_model.RefTrainer` with an `optimizer="sgd"` path
                   (torch.optim.SGD(lr, momentum, nesterov, weight_decay=0)) and a choice of L2 rule

Run as a script, it records tests/golden/optim_sgd.pt from the live reference (utils/optim.py
imported unmodified):

    python tests/sgd_oracle.py

  * `l2`: cal_l2_loss(toy, wd, 'slimmable') and its autograd gradient per parameter, on a toy module
    whose parameters cover every branch of the rule;
  * `nesterov`, `momentum`: 12 steps of the optimizer the reference's get_optimizer(model, FLAGS)
    builds for `optimizer: sgd`, over two parameters: every parameter and momentum buffer after
    every step;
  * `dampening`: the same for torch.optim.SGD(momentum 0.9, dampening 0.5, weight_decay 1e-2),
    which that builder cannot express, with parameter `b` gradless for its first three steps.
"""
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import optim as oo  # noqa: E402
from oracle import torch_model as tm  # noqa: E402

f32 = np.float32
GOLDEN = os.path.join(ROOT, "tests", "golden", "optim_sgd.pt")
REF = os.environ.get("YAMB_REFERENCE", "/root/reference")

# the optimizer section of apps/mobilenet/default.yml
DEFAULT_YML = dict(momentum=0.9, nesterov=True, weight_decay=1e-4, weight_decay_method="slimmable",
                   base_lr=0.5, base_total_batch=1024, label_smoothing=0.0, ema_decay=0.0)

SGD_CASES = {
    # tag: (FLAGS of the reference's get_optimizer, or the torch.optim.SGD kwargs), gradless steps
    "nesterov": dict(flags=dict(lr=0.05, momentum=0.9, nesterov=True), gradless={}),
    "momentum": dict(flags=dict(lr=0.05, momentum=0.9, nesterov=False), gradless={}),
    "dampening": dict(kw=dict(lr=0.05, momentum=0.9, dampening=0.5, weight_decay=1e-2),
                      gradless={"b": (0, 1, 2)}),
}
SGD_SHAPES = {"a": (257,), "b": (5, 7)}
STEPS = 12


def sgd_step(p, g, buf, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False):
    """One torch.optim.SGD.step() of one parameter on flat float32 arrays; `buf` None = the
    parameter has no momentum buffer yet.  Returns (p, buf) (new arrays)."""
    p, g = p.astype(f32), g.astype(f32)
    if weight_decay != 0:                                   # grad = grad.add(param, alpha=wd)
        g = g + f32(weight_decay) * p
    if momentum != 0:
        if buf is None:                                     # buf = grad.detach().clone()
            buf = g.copy()
        else:                                               # buf.mul_(m).add_(grad, alpha=1-d)
            buf = buf.astype(f32) * f32(momentum) + f32(1 - dampening) * g
        if nesterov:                                        # grad = grad.add(buf, alpha=m)
            g = g + f32(momentum) * buf
        else:                                               # grad = buf
            g = buf
    p = p - f32(lr) * g                                     # param.add_(grad, alpha=-lr)
    return p.astype(f32), (buf.astype(f32) if buf is not None else None)


def l2_decay_mask(named_shapes, method="mnas"):
    """Which parameters cal_l2_loss(method) regularises (utils/optim.py:161-200).  'slimmable':
    4-D tensors with shape[1] != 1 and all 2-D tensors (:165-176)."""
    named_shapes = list(named_shapes)
    if method == "mnas":
        return oo.l2_decay_mask(named_shapes)
    if method == "slimmable":
        return {name: (len(s) == 4 and s[1] != 1) or len(s) == 2 for name, s in named_shapes}
    if method == "mnas_no_bias":
        raise NotImplementedError()
    raise ValueError("Unknown weight_decay method: {}".format(method))


l2_grad = oo.l2_grad


def l2_loss_slimmable(model, weight_decay):
    """cal_l2_loss(method='slimmable') (utils/optim.py:165-176)."""
    loss = 0.0
    for p in model.parameters():
        s = p.shape
        if (len(s) == 4 and s[1] != 1) or len(s) == 2:
            loss = loss + weight_decay * (p ** 2).sum()
    return loss * 0.5


L2_LOSS = {"mnas": tm.l2_loss_mnas, "slimmable": l2_loss_slimmable}


class RefTrainer(tm.RefTrainer):
    """The reference's training step (train.py:64-114) with `optimizer: sgd` or `rmsprop` and the
    L2 rule `weight_decay_method`.  The defaults are those of oracle.torch_model.RefTrainer."""

    def __init__(self, model, batch_size_global, optimizer="rmsprop", nesterov=False,
                 dampening=0.0, weight_decay_method="mnas", **kw):
        super().__init__(model, batch_size_global, **kw)
        if optimizer == "sgd":                              # utils/optim.py:262-267
            self.opt = torch.optim.SGD(model.parameters(), lr=self.lr,
                                       momentum=kw.get("momentum", 0.9), dampening=dampening,
                                       nesterov=nesterov, weight_decay=0)
        elif optimizer != "rmsprop":
            raise ValueError(optimizer)
        self.l2_loss = L2_LOSS[weight_decay_method]

    def step(self, x, target):
        model = self.model
        model.train()
        self.opt.zero_grad()                                          # train.py:66
        if self.autocast is not None:
            with torch.autocast(x.device.type, dtype=self.autocast):
                out = model(x).float()
        else:
            out = model(x)
        loss_vec = tm.label_smooth_ce(out, target, self.smoothing)
        _ = loss_vec.tolist()                                         # common.py:71 host sync #1
        _, pred = out.topk(5)
        correct = pred.t().eq(target.view(1, -1).expand_as(pred.t()))
        for k in (1, 5):
            _ = correct[:k].float().sum(0).cpu().numpy()              # common.py:73-79 sync #2
        loss = loss_vec.mean() + self.l2_loss(model, self.wd)         # train.py:68-70
        loss.backward()
        self.opt.step()                                               # train.py:102
        self.global_step += 1
        named = dict(model.named_parameters())
        named.update({n: b for n, b in model.named_buffers()})
        for n in self.ema.shadow:                                     # train.py:109-114
            self.ema(n, named[n], self.global_step)
        return float(loss.detach())


class L2Toy(torch.nn.Module):
    """Parameters covering every branch of the 'slimmable' rule: stem [8,3,3,3], pointwise
    [16,8,1,1], depthwise [16,1,3,3], a one-channel branch's pointwise [8,1,1,1] (AtomNAS widths),
    an SE conv with bias, BatchNorm gamma/beta and the classifier."""

    def __init__(self):
        super().__init__()
        self.stem = torch.nn.Conv2d(3, 8, 3, bias=False)
        self.pw = torch.nn.Conv2d(8, 16, 1, bias=False)
        self.dw = torch.nn.Conv2d(16, 16, 3, groups=16, bias=False)
        self.pw1 = torch.nn.Conv2d(1, 8, 1, bias=False)
        self.se_reduce = torch.nn.Conv2d(16, 4, 1)
        self.bn = torch.nn.BatchNorm2d(16)
        self.classifier = torch.nn.Linear(16, 10)


def load_golden():
    return torch.load(GOLDEN, weights_only=False)


def main():
    sys.path.insert(0, REF)
    warnings.simplefilter("ignore")
    from utils import optim as roptim
    rec = {}
    torch.manual_seed(11)
    toy = L2Toy()
    with torch.no_grad():
        for p in toy.parameters():
            p.normal_(0, 0.5)
    wd = 1e-2
    l2 = roptim.cal_l2_loss(toy, wd, "slimmable")
    l2.backward()
    rec["l2"] = {"wd": wd, "loss": l2.detach().clone(),
                 "params": {k: p.detach().clone() for k, p in toy.named_parameters()},
                 "grads": {k: (p.grad.clone() if p.grad is not None else torch.zeros_like(p))
                           for k, p in toy.named_parameters()}}

    class Flags:
        optimizer = "sgd"

    for tag, case in SGD_CASES.items():
        torch.manual_seed(5)
        params = {k: torch.nn.Parameter(torch.randn(s)) for k, s in SGD_SHAPES.items()}
        model = torch.nn.Module()
        for k, p in params.items():
            model.register_parameter(k, p)
        if "flags" in case:
            fl = Flags()
            for k, v in case["flags"].items():
                setattr(fl, k, v)
            opt = roptim.get_optimizer(model, fl)
            kw = dict(lr=fl.lr, momentum=fl.momentum, nesterov=fl.nesterov)
        else:
            kw = dict(case["kw"])
            opt = torch.optim.SGD(model.parameters(), **kw)
        assert isinstance(opt, torch.optim.SGD)
        out = {"kw": kw, "gradless": case["gradless"], "params": {}}
        seq = {k: {"p0": p.detach().clone(), "grads": [], "has_grad": [], "ps": [], "bufs": [],
                   "has_buf": []} for k, p in params.items()}
        for step in range(STEPS):
            for k, p in params.items():
                gr = torch.randn(p.shape) * (0.5 + 0.1 * step)
                if step in case["gradless"].get(k, ()):
                    p.grad = None
                    seq[k]["grads"].append(torch.zeros_like(p))
                    seq[k]["has_grad"].append(False)
                else:
                    p.grad = gr.clone()
                    seq[k]["grads"].append(gr)
                    seq[k]["has_grad"].append(True)
            opt.step()
            for k, p in params.items():
                buf = opt.state[p].get("momentum_buffer")
                seq[k]["ps"].append(p.detach().clone())
                seq[k]["bufs"].append(buf.clone() if buf is not None else torch.zeros_like(p))
                seq[k]["has_buf"].append(buf is not None)
        for k, s in seq.items():
            out["params"][k] = {"p0": s["p0"], "grads": torch.stack(s["grads"]),
                                "has_grad": torch.tensor(s["has_grad"]),
                                "ps": torch.stack(s["ps"]), "bufs": torch.stack(s["bufs"]),
                                "has_buf": torch.tensor(s["has_buf"])}
        rec[tag] = out
    torch.save(rec, GOLDEN)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    main()
