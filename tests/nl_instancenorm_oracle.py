"""Oracle and fixture generator of the non-local block with `nl_norm: nn.InstanceNorm`.

The norm is nn.InstanceNorm2d(C, affine=True, track_running_stats=True) (reference
models/mobilenet_base.py:149-156, :472-481).  `extract` / `forward` / `backward` restate that
block in plain torch fp32 on top of oracle/ir_block.py, which covers everything up to the
non-local block's input l = BN3(h3) and everything behind its gradient dl:

  training : per (n, c) mean and biased variance over H*W; running statistics
             (1-m)*running + m*mean_n(batch) with each instance's UNBIASED variance, no update when
             momentum is None, num_batches_tracked untouched (torch.nn.functional.instance_norm)
  eval     : the running statistics (a per-channel affine, as BatchNorm)

`quant=True` rounds to bf16 where the CUDA path materialises a tensor: the instance statistics come
from the bf16 h the kernel reads, and dh is rounded where yamb_instance_norm_bwd writes it.

    python tests/nl_instancenorm_oracle.py      # writes tests/golden/blocks_nl_in.pt

runs the LIVE reference (the checkout oracle/make_golden.py uses, YAMB_REFERENCE) with the
AutoNL yml and FLAGS.nl_norm = "nn.InstanceNorm"; only the fixture travels with the repository.

The fixture stores what the reference computed (y, dx, every parameter gradient, the buffers after
the call) but not its inputs: the block's initial state, x and dy come from a seeded recipe
(`_seeded_block`) that this package's modules reproduce bit for bit, and the fp64 sum
of every initial state tensor is stored so that `load_golden` notices if they ever do not.
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ir_block as ob  # noqa: E402

# the four kinds of non-local block of tests/golden/blocks_nl.pt (both association orders of the
# reference's MAC test, a skip connection, SE, nl_s = 2 on an odd map, stride 2; the odd-map case at
# its shape there, the others at smaller widths and maps that keep the fixture small), plus an
# AutoNL-L-like 7x7 map with nl_c = 1/8
CASES = [
    ("in_B_res", "InvertedResidualChannelsFused", (24, 24, 1, [48], [3], True), "nn.Swish",
     {"se_ratio": 0.25, "nl_c": 0.25, "nl_s": 1}, (2, 24, 8, 8)),
    ("in_A_small_map", "InvertedResidualChannelsFused", (48, 48, 1, [48], [3], True), "nn.Swish",
     {"nl_c": 0.25, "nl_s": 1}, (2, 48, 4, 4)),
    ("in_sub2_odd_map", "InvertedResidualChannelsFused", (40, 40, 1, [120], [5], True), "nn.Swish",
     {"se_ratio": 0.25, "nl_c": 0.25, "nl_s": 2}, (2, 40, 7, 7)),
    ("in_s2_nores", "InvertedResidualChannelsFused", (16, 24, 2, [48], [5], True), "nn.ReLU6",
     {"nl_c": 0.25, "nl_s": 2}, (2, 16, 8, 8)),
    ("in_autonl_7x7", "InvertedResidualChannelsFused", (32, 32, 1, [64], [3], True), "nn.Swish",
     {"se_ratio": 0.25, "nl_c": 0.125, "nl_s": 1}, (2, 32, 7, 7)),
]
GOLDEN = "blocks_nl_in.pt"


def extract(block):
    """(cfg, P) as oracle.ir_block.extract, with the InstanceNorm's tensors under bn4_*."""
    nl = block.nl_op
    if not isinstance(nl.bn, torch.nn.InstanceNorm2d):
        raise ValueError("not an InstanceNorm non-local block")
    block.nl_op = torch.nn.Identity()
    try:
        cfg, P = ob.extract(block)
    finally:
        block.nl_op = nl
    norm = nl.bn
    P["w_nl"] = nl.depthwise_conv.weight.detach()[:, 0]
    P["bn4_g"], P["bn4_b"] = norm.weight.detach(), norm.bias.detach()
    P["bn4_rm"], P["bn4_rv"] = norm.running_mean, norm.running_var
    P["bn4_eps"], P["bn4_momentum"] = norm.eps, norm.momentum
    return cfg._replace(nl_c=nl.nl_c, nl_s=nl.nl_s), P


def _inner(cfg):
    """The block up to l = BN3(h3): no non-local block, no skip connection."""
    return cfg._replace(nl_c=0, nl_s=1, residual=False)


def forward(x, cfg, P, training=True, quant=False):
    q = bool(quant)
    l, S = ob.forward(x, _inner(cfg), P, training=training, quant=quant)   # _rnd(BN3(h3))
    N, C, H, W = l.shape
    c, s_ = int(cfg.nl_c * C), cfg.nl_s
    lr = l[:, :, ::s_, ::s_]
    Fm = torch.einsum("nihw,njhw->nij", lr[:, :c], lr)
    f = ob._rnd(torch.einsum("nij,nihw->njhw", Fm, l[:, :c]) / H * W, q)    # sic (f/H)*W
    hn = ob._rnd(F.conv2d(f, P["w_nl"][:, None], None, 1, 1, 1, C), q)
    g, b, eps = P["bn4_g"], P["bn4_b"], P["bn4_eps"]
    if training:
        mean = hn.mean((2, 3))
        var = hn.var((2, 3), unbiased=False)
        invstd = torch.rsqrt(var + eps)
        m = 0.0 if P["bn4_momentum"] is None else P["bn4_momentum"]
        hw = H * W
        S["bn4_rm_after"] = (1 - m) * P["bn4_rm"] + m * mean.mean(0)
        S["bn4_rv_after"] = (1 - m) * P["bn4_rv"] + m * (var * (hw / (hw - 1))).mean(0)
    else:
        mean = P["bn4_rm"][None].expand(N, C)
        invstd = torch.rsqrt(P["bn4_rv"] + eps)[None].expand(N, C)
    xhat = (hn - mean[:, :, None, None]) * invstd[:, :, None, None]
    y = g[None, :, None, None] * xhat + b[None, :, None, None] + l
    if cfg.residual:
        y = y + S["x"]
    S.update(nl_l=l, nl_F=Fm, nl_f=f, nl_hn=hn, bn4_mean=mean, bn4_invstd=invstd)
    return ob._rnd(y, q), S


def backward(dy, cfg, P, S, training=True, quant=False):
    q = quant
    dy = ob._rnd(dy, q)
    l, Fm, f, hn = S["nl_l"], S["nl_F"], S["nl_f"], S["nl_hn"]
    N, C, H, W = l.shape
    c, s_ = int(cfg.nl_c * C), cfg.nl_s
    sc = float(W) / float(H)
    mean, invstd = S["bn4_mean"][:, :, None, None], S["bn4_invstd"][:, :, None, None]
    xhat = (hn - mean) * invstd
    G = {}
    sdy = dy.sum((2, 3), keepdim=True)
    sdx = (dy * xhat).sum((2, 3), keepdim=True)
    G["bn4_g"], G["bn4_b"] = sdx.sum((0, 2, 3)), sdy.sum((0, 2, 3))
    a = P["bn4_g"][None, :, None, None] * invstd
    dhn = a * (dy - sdy / (H * W) - xhat * sdx / (H * W)) if training else a * dy
    dhn = ob._rnd(dhn, q)
    # the rest of the non-local backward, as oracle.ir_block.backward
    df = ob._rnd(torch.nn.grad.conv2d_input(f.shape, P["w_nl"][:, None], dhn, 1, 1, 1, C), q)
    G["w_nl"] = torch.nn.grad.conv2d_weight(f, (C, 1, 3, 3), dhn, 1, 1, 1, C)[:, 0]
    dF = torch.einsum("nihw,njhw->nij", l[:, :c], df) * sc
    dl = dy.clone()
    dl[:, :c] += torch.einsum("njhw,nij->nihw", df, Fm) * sc
    dl = ob._rnd(dl, q)
    lr = l[:, :, ::s_, ::s_]
    dl[:, :c, ::s_, ::s_] = ob._rnd(dl[:, :c, ::s_, ::s_] +
                                    torch.einsum("njhw,nij->nihw", lr, dF), q)
    dl[:, :, ::s_, ::s_] = ob._rnd(dl[:, :, ::s_, ::s_] +
                                   torch.einsum("nihw,nij->njhw", lr[:, :c], dF), q)
    dx, G2 = ob.backward(dl, _inner(cfg), P, S, training=training, quant=quant)
    G.update(G2)
    if cfg.residual:
        dx = ob._rnd(dx + dy, q)
    return dx, G


def named_grads(cfg, G):
    """Merged-layout gradients of a single-branch fused block -> {parameter name: gradient}."""
    got = {"depth_ops.0.1.0.weight": G["w_dw"][0], "depth_ops.0.1.1.weight": G["bn2_g"],
           "depth_ops.0.1.1.bias": G["bn2_b"], "project_conv.0.weight": G["w_proj"],
           "project_conv.1.weight": G["bn3_g"], "project_conv.1.bias": G["bn3_b"],
           "nl_op.depthwise_conv.weight": G["w_nl"], "nl_op.bn.weight": G["bn4_g"],
           "nl_op.bn.bias": G["bn4_b"]}
    if cfg.expand:
        got.update({"expand_conv.0.weight": G["w_exp"], "expand_conv.1.weight": G["bn1_g"],
                    "expand_conv.1.bias": G["bn1_b"]})
    for k, name in (("se_wr", "se_op.se_reduce.weight"), ("se_br", "se_op.se_reduce.bias"),
                    ("se_we", "se_op.se_expand.weight"), ("se_be", "se_op.se_expand.bias")):
        if k in G:
            got[name] = G[k]
    return got


def randomise_norms(block, g):
    """Non-trivial affine parameters and running statistics of every BatchNorm and of the
    InstanceNorm (both start at gamma = beta = 0 / running statistics 0 and 1)."""
    for m in block.modules():
        if isinstance(m, (torch.nn.BatchNorm2d, torch.nn.InstanceNorm2d)):
            m.weight.data.uniform_(0.5, 1.5, generator=g)
            m.bias.data.normal_(0, 0.3, generator=g)
            m.running_mean.normal_(0, 0.2, generator=g)
            m.running_var.uniform_(0.5, 1.5, generator=g)


BN_KW = {"momentum": 0.01, "eps": 1e-3}


def _seeded_block(mb, case, replace_norm=False):
    """The block of a case with its seeded initial state (init_weights_mnas, then non-trivial
    norms) and the generator that then draws x and the dy of train and eval, in that order.
    `replace_norm`: install the InstanceNorm explicitly (this package, without the reference's
    FLAGS) before initialising; neither norm's construction consumes random numbers."""
    name, cls, args, act, extra, xshape = case
    torch.manual_seed(1995)
    blk = getattr(mb, cls)(*args, active_fn=mb.get_active_fn(act), batch_norm_kwargs=BN_KW,
                           **extra)
    if replace_norm:
        blk.nl_op.bn = mb.get_nl_norm_fn("nn.InstanceNorm")(blk.nl_op.n_feature, **BN_KW)
    blk.apply(mb.init_weights_mnas)
    assert isinstance(blk.nl_op.bn, torch.nn.InstanceNorm2d)
    g = torch.Generator().manual_seed(7)
    randomise_norms(blk, g)
    return blk, g


def _state_sums(state):
    return {k: float(v.double().sum()) for k, v in state.items()}


def _pack(tensors):
    """{name: tensor} -> one flat fp32 tensor of the floating-point tensors + their (name, shape)
    (one storage instead of an archive entry per tensor), integer scalars as Python ints."""
    fl = [k for k, v in tensors.items() if v.is_floating_point()]
    return {"entries": [(k, tuple(tensors[k].shape)) for k in fl],
            "flat": torch.cat([tensors[k].detach().float().reshape(-1) for k in fl]),
            "ints": {k: int(v) for k, v in tensors.items() if not v.is_floating_point()}}


def _unpack(packed):
    out, o = {}, 0
    for k, shape in packed["entries"]:
        n = 1
        for d in shape:
            n *= d
        out[k] = packed["flat"][o:o + n].reshape(shape).clone()
        o += n
    out.update({k: torch.tensor(v) for k, v in packed["ints"].items()})
    return out


def load_golden():
    """{case: record} of tests/golden/blocks_nl_in.pt with the inputs rebuilt from the seeded
    recipe: "state", "x", and per mode "dy", "y", "dx", "grads", "state_after"."""
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    stored = torch.load(os.path.join(ROOT, "tests", "golden", GOLDEN), weights_only=False)
    out = {}
    for case in CASES:
        name, cls, args, act, extra, xshape = case
        rec = stored[name]
        blk, g = _seeded_block(mb, case, replace_norm=True)
        state = {k: v.clone() for k, v in blk.state_dict().items()}
        sums = _state_sums(state)
        if sums != rec["state_sums"]:
            raise RuntimeError("%s: the seeded initial state differs from the reference's" % name)
        full = {"cls": cls, "args": args, "act": act, "extra": extra, "bn": BN_KW, "state": state,
                "x": torch.randn(*xshape, generator=g)}
        for mode in ("train", "eval"):
            t = _unpack(rec[mode])
            r = {"y": t.pop("y"), "dx": t.pop("dx")}
            r["dy"] = torch.randn(r["y"].shape, generator=g)
            r["grads"] = {k[len("grad."):]: v for k, v in t.items() if k.startswith("grad.")}
            after = dict(state)
            after.update({k[len("buffer."):]: v for k, v in t.items() if k.startswith("buffer.")})
            r["state_after"] = after
            full[mode] = r
        out[name] = full
    return out


def main():
    """tests/golden/blocks_nl_in.pt from the live reference: its Nonlocal reads FLAGS.nl_norm
    (models/mobilenet_base.py:151), so load the AutoNL yml as its train.py does and set it."""
    from oracle.make_golden import REF as ref
    os.environ.setdefault("ARNOLD_OUTPUT", "/tmp/yamb_out")
    os.environ.setdefault("DATA_LMDB", "/tmp/yamb_lmdb")
    sys.argv = ["nl_instancenorm_oracle", "app:" + os.path.join(ref, "apps/searched/autonl/autonl_l.yml")]
    sys.path.insert(0, ref)
    cwd = os.getcwd()
    os.chdir(ref)
    import logging
    import warnings
    from utils.config import FLAGS
    import models.mobilenet_base as mb
    logging.disable(logging.CRITICAL)
    os.chdir(cwd)
    warnings.simplefilter("ignore")
    FLAGS.nl_norm = "nn.InstanceNorm"
    blocks = {}
    for case in CASES:
        blk, g = _seeded_block(mb, case)
        state0 = {k: v.clone() for k, v in blk.state_dict().items()}
        x = torch.randn(*case[5], generator=g)
        rec = {"state_sums": _state_sums(state0)}
        for mode in ("train", "eval"):
            blk.load_state_dict(state0)
            blk.train(mode == "train")
            blk.zero_grad()
            xi = x.clone().requires_grad_(True)
            y = blk(xi)
            dy = torch.randn(y.shape, generator=g)
            y.backward(dy)
            t = {"y": y, "dx": xi.grad}
            t.update({"grad." + k: p.grad for k, p in blk.named_parameters()})
            t.update({"buffer." + k: v for k, v in blk.named_buffers()})
            rec[mode] = _pack(t)
        blocks[case[0]] = rec
    out = os.path.join(ROOT, "tests", "golden", GOLDEN)
    torch.save(blocks, out)
    print(GOLDEN, os.path.getsize(out), "bytes")


def build_block(rec):
    """This package's block of a `load_golden` record (nl_norm given explicitly: no FLAGS
    needed)."""
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    blk = getattr(mb, rec["cls"])(*rec["args"], active_fn=mb.get_active_fn(rec["act"]),
                                  batch_norm_kwargs=rec["bn"], **rec["extra"])
    nl = blk.nl_op
    nl.bn = mb.get_nl_norm_fn("nn.InstanceNorm")(nl.n_feature, **rec["bn"])
    blk.load_state_dict(rec["state"])
    return blk


if __name__ == "__main__":
    main()
