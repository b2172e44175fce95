"""ORACLE — test infrastructure only (never imported by the product path).

CPU restatement, in plain torch fp32 tensor ops, of the reference's inverted-residual block
forward AND hand-derived backward:

  InvertedResidualChannels.forward        /root/reference/models/mobilenet_base.py:446-451
  InvertedResidualChannelsFused.forward   /root/reference/models/mobilenet_base.py:330-342
  ConvBNReLU                              /root/reference/models/mobilenet_base.py:181-203
  SqueezeAndExcitation.forward            /root/reference/models/mobilenet_base.py:110-113
  Nonlocal.forward                        /root/reference/models/mobilenet_base.py:158-173
  activations                             /root/reference/models/mobilenet_base.py:70-88, 461-469

The arithmetic of the reference lives in PyTorch (torch.nn.functional conv2d / batch_norm,
`requirements.txt:1`); this file restates the *module graph* on top of the same primitives and
adds the explicit backward formulas the CUDA kernels implement, so that each intermediate
(h1, h2, h3, BN statistics, dz, dh, every parameter gradient) can be compared.

Pinning: the reference's own tests hold no numerical fixture for this path (SURVEY.md §8c:
"parity unpinned" upstream), so the oracle is pinned against the LIVE reference modules imported
from /root/reference (oracle/make_golden.py -> tests/golden/*.pt, tests/test_oracle_vs_golden.py)
and its backward against torch.autograd of the reference modules.

`quant=True` additionally rounds to bf16 at exactly the points where the CUDA path materialises a
bf16 tensor (activations in HBM, MMA operands); that mode is what the kernels are compared with
at tight tolerance, while quant=False is what is compared with the reference.
"""
import collections

import torch
import torch.nn.functional as F

ACTS = ("none", "relu", "relu6", "swish", "hswish")


def act_fwd(z, act):
    if act == "relu":
        return torch.relu(z)
    if act == "relu6":
        return torch.clamp(z, 0.0, 6.0)
    if act == "swish":  # mobilenet_base.py:77-78
        return z * torch.sigmoid(z)
    if act == "hswish":  # mobilenet_base.py:87-88
        return z * torch.clamp(z + 3.0, 0.0, 6.0) / 6.0
    return z


def act_bwd(z, act):
    """d act(z) / dz (sub-gradient 0 at the kinks, as torch does)."""
    if act == "relu":
        return (z > 0).to(z.dtype)
    if act == "relu6":
        return ((z > 0) & (z < 6)).to(z.dtype)
    if act == "swish":
        s = torch.sigmoid(z)
        return s * (1 + z * (1 - s))
    if act == "hswish":
        return torch.where(z <= -3, torch.zeros_like(z),
                           torch.where(z >= 3, torch.ones_like(z), (2 * z + 3) / 6))
    return torch.ones_like(z)


def _rnd(t, quant):
    return t.to(torch.bfloat16).to(torch.float32) if quant else t


def act_name(active_fn):
    """Map the reference's zero-arg activation factory (get_active_fn, :461-469) to a name."""
    m = active_fn() if callable(active_fn) and not isinstance(active_fn, torch.nn.Module) \
        else active_fn
    n = type(m).__name__
    return {"ReLU": "relu", "ReLU6": "relu6", "Swish": "swish", "HSwish": "hswish",
            "Identity": "none"}[n]


BlockCfg = collections.namedtuple(
    "BlockCfg", "inp oup stride channels kernel_sizes expand act eps momentum residual se_hidden "
                "nl_c nl_s", defaults=(0, 1))


def extract(block):
    """Canonical (merged) parameters of a reference-compatible block module.

    Works on both packings (they are the same function, SURVEY.md §0): per-branch tensors of
    `InvertedResidualChannels` (ops.b.*) are concatenated along the hidden dimension exactly as
    `InvertedResidualChannelsFused` stores them.
    Returns (cfg, P) with P a dict of tensors (references to the module's tensors where possible).
    """
    fused = hasattr(block, "expand_conv")
    chans, ks = list(block.channels), list(block.kernel_sizes)
    P = {}

    def bn_pack(prefix, bns):
        P[prefix + "_g"] = torch.cat([b.weight.detach() for b in bns])
        P[prefix + "_b"] = torch.cat([b.bias.detach() for b in bns])
        P[prefix + "_rm"] = torch.cat([b.running_mean for b in bns])
        P[prefix + "_rv"] = torch.cat([b.running_var for b in bns])

    if fused:
        if block.expand:
            P["w_exp"] = block.expand_conv[0].weight.detach().flatten(1)
            bn_pack("bn1", [block.expand_conv[1]])
        dws = [list(op.children())[-1] for op in block.depth_ops]
        P["w_dw"] = [d[0].weight.detach()[:, 0] for d in dws]
        bn_pack("bn2", [d[1] for d in dws])
        P["w_proj"] = block.project_conv[0].weight.detach().flatten(1)
        bn3 = block.project_conv[1]
        se = block.se_op if hasattr(block.se_op, "se_reduce") else None
        if se is not None:
            P["se_wr"] = se.se_reduce.weight.detach().flatten(1)
            P["se_br"] = se.se_reduce.bias.detach()
            P["se_we"] = se.se_expand.weight.detach().flatten(1)
            P["se_be"] = se.se_expand.bias.detach()
        nl = block.nl_op if type(block.nl_op).__name__ != "Identity" else None
        if nl is not None:
            if not isinstance(nl.bn, torch.nn.BatchNorm2d):
                raise NotImplementedError("oracle: non-local block with a non-BatchNorm nl_norm")
            P["w_nl"] = nl.depthwise_conv.weight.detach()[:, 0]
            bn_pack("bn4", [nl.bn])
        bn_any = bn3
    else:
        se = None
        nl = None
        if block.expand:
            P["w_exp"] = torch.cat([op[0][0].weight.detach().flatten(1) for op in block.ops])
            bn_pack("bn1", [op[0][1] for op in block.ops])
            dws = [op[1] for op in block.ops]
            P["w_proj"] = torch.cat([op[2].weight.detach().flatten(1) for op in block.ops], 1)
        else:
            dws = [op[0] for op in block.ops]
            P["w_proj"] = torch.cat([op[1].weight.detach().flatten(1) for op in block.ops], 1)
        P["w_dw"] = [d[0].weight.detach()[:, 0] for d in dws]
        bn_pack("bn2", [d[1] for d in dws])
        bn_any = block.pw_bn
    bn_pack("bn3", [bn_any])
    if not block.expand and not fused and len(chans) > 1:
        # every branch consumes the whole input (mobilenet_base.py:396-402): hidden = inp per branch
        pass
    cfg = BlockCfg(inp=block.input_dim, oup=block.output_dim, stride=block.stride,
                   channels=chans, kernel_sizes=ks, expand=bool(block.expand),
                   act=act_name(block.active_fn), eps=bn_any.eps, momentum=bn_any.momentum,
                   residual=bool(block.use_res_connect),
                   se_hidden=(P["se_wr"].shape[0] if se is not None else 0),
                   nl_c=(nl.nl_c if nl is not None else 0), nl_s=(nl.nl_s if nl is not None else 1))
    return cfg, P


def _bn_train(h, g, b, eps):
    """Batch statistics over (N,H,W) — biased variance for normalisation (nn.BatchNorm2d)."""
    mean = h.mean((0, 2, 3))
    var = h.var((0, 2, 3), unbiased=False)
    invstd = torch.rsqrt(var + eps)
    scale = g * invstd
    shift = b - mean * scale
    return scale, shift, mean, invstd, var


def bn_running_update(rm, rv, mean, var, count, momentum, nbt):
    """running = (1-m)*running + m*batch with UNBIASED variance; momentum=None -> 1/nbt."""
    nbt = nbt + 1
    m = (1.0 / nbt) if momentum is None else momentum
    unb = var * (count / max(count - 1, 1))
    return (1 - m) * rm + m * mean, (1 - m) * rv + m * unb, nbt


def _dw(a, w_list, channels, stride):
    outs, c0 = [], 0
    for w, c in zip(w_list, channels):
        k = w.shape[-1]
        outs.append(F.conv2d(a[:, c0:c0 + c], w[:, None], None, stride, (k - 1) // 2, 1, c))
        c0 += c
    return outs[0] if len(outs) == 1 else torch.cat(outs, 1)


def forward(x, cfg, P, training=True, quant=False):
    """y, saved.  x: [N,Cin,H,W] fp32.  `saved` holds every intermediate the backward needs plus
    the batch statistics (for the running-stat check)."""
    q = bool(quant)
    # quant="fused": rounding points of the one-launch eval kernel (csrc/block_eval.cu), which keeps
    # the raw convolution outputs h1 / h2 / h3 in fp32 (registers) and rounds only the
    # activations it stages as tensor-core operands and the block output
    qr = quant is True
    S = {}
    x = _rnd(x, q)
    S["x"] = x
    chid = sum(cfg.channels)
    M_in = x.shape[0] * x.shape[2] * x.shape[3]

    def bn(h, pfx, stat_src=None):
        if training:
            scale, shift, mean, invstd, var = _bn_train(h if stat_src is None else stat_src,
                                                        P[pfx + "_g"], P[pfx + "_b"], cfg.eps)
            S[pfx + "_mean"], S[pfx + "_invstd"], S[pfx + "_var"] = mean, invstd, var
        else:
            invstd = torch.rsqrt(P[pfx + "_rv"] + cfg.eps)
            scale = P[pfx + "_g"] * invstd
            shift = P[pfx + "_b"] - P[pfx + "_rm"] * scale
            S[pfx + "_mean"], S[pfx + "_invstd"] = P[pfx + "_rm"], invstd
        S[pfx + "_scale"], S[pfx + "_shift"] = scale, shift
        return h * scale[None, :, None, None] + shift[None, :, None, None]

    if cfg.expand:
        h1 = _rnd(F.conv2d(x, _rnd(P["w_exp"], q)[:, :, None, None]), qr)
        S["h1"] = h1
        a1 = _rnd(act_fwd(bn(h1, "bn1"), cfg.act), q)  # staged in shared memory as bf16
    else:
        # unfused, expand=False: each branch sees the whole input (hidden == inp)
        a1 = x if len(cfg.channels) == 1 else torch.cat([x] * len(cfg.channels), 1)
    S["a1"] = a1
    h2_acc = _dw(a1, P["w_dw"], cfg.channels, cfg.stride)
    h2 = _rnd(h2_acc, qr)
    S["h2"] = h2
    # the depthwise kernel takes the BN2 statistics from its fp32 accumulators, not from the
    # bf16 values it stores (a zero-mean 2^-9 rounding noise apart they are the same numbers)
    a2 = _rnd(act_fwd(bn(h2, "bn2", h2_acc), cfg.act), q)  # MMA operand -> bf16
    S["a2"] = a2
    if cfg.se_hidden:
        s = a2.mean((2, 3))
        u = s @ P["se_wr"].t() + P["se_br"]
        v = act_fwd(u, cfg.act)
        t = v @ P["se_we"].t() + P["se_be"]
        gate = torch.sigmoid(t)
        S.update(se_s=s, se_u=u, se_v=v, se_gate=gate)
        a2 = _rnd(a2 * gate[:, :, None, None], q)
        S["a2s"] = a2
    h3 = _rnd(F.conv2d(a2, _rnd(P["w_proj"], q)[:, :, None, None]), qr)
    S["h3"] = h3
    y = bn(h3, "bn3")
    if cfg.nl_c > 0:
        # Nonlocal.forward (:158-173).  The reference picks (theta phi^T) g or theta (phi^T g) by
        # a MAC count (:164-170) — one sum, two association orders; the channel-matrix order is
        # restated here (it is what the CUDA path always uses).
        l = _rnd(y, q)                                   # BN3 output, materialised bf16
        n_, C_, H_, W_ = l.shape
        c, s_ = int(cfg.nl_c * C_), cfg.nl_s
        lr = l[:, :, ::s_, ::s_]
        Fm = torch.einsum("nihw,njhw->nij", lr[:, :c], lr)             # phi^T g, fp32
        f = _rnd(torch.einsum("nij,nihw->njhw", Fm, l[:, :c]) / H_ * W_, q)   # sic: (f/H)*W, :171
        hn_acc = F.conv2d(f, P["w_nl"][:, None], None, 1, 1, 1, C_)
        hn = _rnd(hn_acc, q)
        S.update(nl_l=l, nl_F=Fm, nl_f=f, nl_hn=hn)
        y = bn(hn, "bn4", hn_acc) + l
    if cfg.residual:
        y = y + x
    y = _rnd(y, q)
    S["count_in"] = M_in
    S["count_out"] = h3.shape[0] * h3.shape[2] * h3.shape[3]
    assert h2.shape[1] == chid
    return y, S


def _bn_bwd(dz, h, mean, invstd, g, training, dz_stats=None):
    """dgamma, dbeta, dh for z = g*xhat + b, xhat = (h-mean)*invstd.  `dz_stats`: the values the
    sums are taken from when they differ from the (bf16-rounded) dz that is propagated."""
    xhat = (h - mean[None, :, None, None]) * invstd[None, :, None, None]
    ds = dz if dz_stats is None else dz_stats
    dg = (ds * xhat).sum((0, 2, 3))
    db = ds.sum((0, 2, 3))
    sc = (g * invstd)[None, :, None, None]
    if training:
        M = dz.shape[0] * dz.shape[2] * dz.shape[3]
        dh = sc * (dz - (db / M)[None, :, None, None] - xhat * (dg / M)[None, :, None, None])
    else:
        dh = sc * dz
    return dg, db, dh


def backward(dy, cfg, P, S, training=True, quant=False):
    """dx and a dict of parameter gradients (merged layout, see `extract`)."""
    q = quant
    G = {}
    dy = _rnd(dy, q)
    x = S["x"]
    dy_in = dy                                           # what the skip connection carries back
    if cfg.nl_c > 0:
        # --- autograd of Nonlocal.forward: bn4 -> depthwise 3x3 -> the two products; `+ l` ---
        l, Fm, f, hn = S["nl_l"], S["nl_F"], S["nl_f"], S["nl_hn"]
        n_, C_, H_, W_ = l.shape
        c, s_ = int(cfg.nl_c * C_), cfg.nl_s
        sc = float(W_) / float(H_)
        G["bn4_g"], G["bn4_b"], dhn = _bn_bwd(dy, hn, S["bn4_mean"], S["bn4_invstd"], P["bn4_g"],
                                              training)
        dhn = _rnd(dhn, q)                               # staged bf16 by the depthwise backward
        df = _rnd(torch.nn.grad.conv2d_input(f.shape, P["w_nl"][:, None], dhn, 1, 1, 1, C_), q)
        G["w_nl"] = torch.nn.grad.conv2d_weight(f, (C_, 1, 3, 3), dhn, 1, 1, 1, C_)[:, 0]
        dF = torch.einsum("nihw,njhw->nij", l[:, :c], df) * sc
        dl = dy.clone()
        dl[:, :c] += torch.einsum("njhw,nij->nihw", df, Fm) * sc           # dtheta
        dl = _rnd(dl, q)
        lr = l[:, :, ::s_, ::s_]
        dl[:, :c, ::s_, ::s_] = _rnd(dl[:, :c, ::s_, ::s_] +
                                     torch.einsum("njhw,nij->nihw", lr, dF), q)        # dphi
        dl[:, :, ::s_, ::s_] = _rnd(dl[:, :, ::s_, ::s_] +
                                    torch.einsum("nihw,nij->njhw", lr[:, :c], dF), q)  # dg
        dy = dl
    # --- BN3 (no activation) ---
    G["bn3_g"], G["bn3_b"], dh3 = _bn_bwd(dy, S["h3"], S["bn3_mean"], S["bn3_invstd"], P["bn3_g"],
                                          training)
    dh3 = _rnd(dh3, q)  # materialised bf16 (MMA operand)
    # --- project 1x1 ---
    a2_in = S["a2s"] if cfg.se_hidden else S["a2"]
    wp = _rnd(P["w_proj"], q)
    G["w_proj"] = torch.einsum("nohw,nchw->oc", dh3, a2_in)
    da2 = torch.einsum("nohw,oc->nchw", dh3, wp)
    if cfg.se_hidden:
        da2 = _rnd(da2, q)  # the CUDA path materialises d(a2*gate) in bf16 before the SE backward
        gate, a2 = S["se_gate"], S["a2"]
        hw = a2.shape[2] * a2.shape[3]
        dgate = (da2 * a2).sum((2, 3))
        dt = dgate * gate * (1 - gate)
        G["se_we"] = dt.t() @ S["se_v"]
        G["se_be"] = dt.sum(0)
        dv = dt @ P["se_we"]
        du = dv * act_bwd(S["se_u"], cfg.act)
        G["se_wr"] = du.t() @ S["se_s"]
        G["se_br"] = du.sum(0)
        ds = du @ P["se_wr"]
        da2 = da2 * gate[:, :, None, None] + (ds / hw)[:, :, None, None]
    # --- BN2 + act ---
    z2 = S["h2"] * S["bn2_scale"][None, :, None, None] + S["bn2_shift"][None, :, None, None]
    dz2 = _rnd(da2 * act_bwd(z2, cfg.act), q)  # materialised bf16
    G["bn2_g"], G["bn2_b"], dh2 = _bn_bwd(dz2, S["h2"], S["bn2_mean"], S["bn2_invstd"], P["bn2_g"],
                                          training)
    dh2 = _rnd(dh2, q)  # staged in shared memory as bf16 by the depthwise backward
    # --- depthwise k x k ---
    a1 = S["a1"]
    da1_parts, G["w_dw"], c0 = [], [], 0
    for w, c in zip(P["w_dw"], cfg.channels):
        k = w.shape[-1]
        pad = (k - 1) // 2
        dh2_b = dh2[:, c0:c0 + c]
        a1_b = a1[:, c0:c0 + c]
        da1_parts.append(torch.nn.grad.conv2d_input(a1_b.shape, w[:, None], dh2_b, cfg.stride,
                                                    pad, 1, c))
        G["w_dw"].append(torch.nn.grad.conv2d_weight(a1_b, (c, 1, k, k), dh2_b, cfg.stride, pad,
                                                     1, c)[:, 0])
        c0 += c
    da1 = da1_parts[0] if len(da1_parts) == 1 else torch.cat(da1_parts, 1)
    if cfg.expand:
        # --- BN1 + act ---
        z1 = S["h1"] * S["bn1_scale"][None, :, None, None] + S["bn1_shift"][None, :, None, None]
        dz1_acc = da1 * act_bwd(z1, cfg.act)
        dz1 = _rnd(dz1_acc, q)  # materialised bf16; the depthwise kernel sums its fp32 values
        G["bn1_g"], G["bn1_b"], dh1 = _bn_bwd(dz1, S["h1"], S["bn1_mean"], S["bn1_invstd"],
                                              P["bn1_g"], training, dz1_acc)
        dh1 = _rnd(dh1, q)  # MMA operand
        we = _rnd(P["w_exp"], q)
        G["w_exp"] = torch.einsum("nohw,nchw->oc", dh1, x)
        dx = torch.einsum("nohw,oc->nchw", dh1, we)
    else:
        nb = len(cfg.channels)
        dx = da1 if nb == 1 else sum(da1.chunk(nb, 1))
    if cfg.residual:
        dx = dx + dy_in
    return _rnd(dx, q), G
