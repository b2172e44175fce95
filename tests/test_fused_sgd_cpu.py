"""CPU: the SGD recipe (`optimizer: sgd`, `weight_decay_method: slimmable`).

The SGD oracle (tests/sgd_oracle.py) against the live reference's records
(tests/golden/optim_sgd.pt), the 'slimmable' and 'mnas' L2 masks of flat_arena.l2_mask, the C ABI of
`yamb_sgd_step` and the constructor contract of fused_sgd.SGD against torch.optim.SGD."""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

import sgd_oracle as so
from _cfg import build_from_cfg, load_cfgs


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


@pytest.fixture(scope="module")
def golden():
    return so.load_golden()


@pytest.mark.parametrize("tag", list(so.SGD_CASES))
def test_oracle_sgd_step_vs_reference(golden, tag):
    rec = golden[tag]
    kw = rec["kw"]
    for name, s in rec["params"].items():
        p = s["p0"].numpy().ravel()
        buf = None
        for i in range(s["grads"].shape[0]):
            if bool(s["has_grad"][i]):
                p, buf = so.sgd_step(p, s["grads"][i].numpy().ravel(), buf, **kw)
            assert _rel(p, s["ps"][i].numpy().ravel()) <= 1e-6, (tag, name, i)
            assert (buf is not None) == bool(s["has_buf"][i]), (tag, name, i)
            if buf is not None:
                assert _rel(buf, s["bufs"][i].numpy().ravel()) <= 1e-6, (tag, name, i)
    if tag == "dampening":    # parameter b had no gradient for its first three steps
        b = rec["params"]["b"]
        assert not bool(b["has_buf"][2]) and bool(b["has_buf"][3])
        assert torch.equal(b["ps"][2], b["p0"])


def test_slimmable_mask_and_l2_grad_vs_reference(golden):
    from yet_another_mobilenet_series_b200.flat_arena import l2_mask
    rec = golden["l2"]
    toy = so.L2Toy()
    named = list(toy.named_parameters())
    assert [k for k, _ in named] == list(rec["params"])
    mask = l2_mask(named, "slimmable")
    omask = so.l2_decay_mask([(k, tuple(p.shape)) for k, p in named], "slimmable")
    assert mask == omask
    for k, p in rec["params"].items():
        want = rec["grads"][k].numpy()
        if mask[k]:
            assert _rel(so.l2_grad(p.numpy(), rec["wd"]), want) <= 1e-6, k
        else:
            assert not want.any(), k       # the reference's gradient is exactly zero
    # the rule is one of shape: the one-channel pointwise and every 1-D tensor are not decayed,
    # the stem and the SE conv weight are
    assert mask["pw1.weight"] is False and mask["classifier.bias"] is False
    assert mask["dw.weight"] is False and mask["se_reduce.bias"] is False
    assert mask["bn.weight"] is False and mask["bn.bias"] is False
    assert mask["stem.weight"] and mask["pw.weight"] and mask["se_reduce.weight"]
    assert mask["classifier.weight"]
    toy.load_state_dict(rec["params"], strict=False)
    loss = so.l2_loss_slimmable(toy, rec["wd"]).detach()
    assert abs(float(loss) - float(rec["loss"])) <= 1e-6 * float(rec["loss"])


@pytest.mark.parametrize("name", sorted(load_cfgs()))
def test_mnas_mask_unchanged_on_configs(name):
    from oracle import optim as oo
    from yet_another_mobilenet_series_b200.flat_arena import l2_mask
    from yet_another_mobilenet_series_b200.fused_rmsprop import mnas_l2_mask
    model, _ = build_from_cfg(name)
    named = list(model.named_parameters())
    want = oo.l2_decay_mask([(k, tuple(p.shape)) for k, p in named])
    assert mnas_l2_mask(named) == want
    assert l2_mask(named, "mnas") == want
    assert sum(want.values()) > 0 and not all(want.values())


def test_l2_mask_errors():
    from yet_another_mobilenet_series_b200.flat_arena import l2_mask
    from yet_another_mobilenet_series_b200.fused_rmsprop import RMSprop
    from yet_another_mobilenet_series_b200.fused_sgd import SGD
    m = nn.Linear(3, 2)
    for opt in (SGD(m.parameters(), lr=0.1), RMSprop(m.parameters(), lr=0.1)):
        with pytest.raises(NotImplementedError):
            opt.fold_l2(1e-4, m.named_parameters(), "mnas_no_bias")
        with pytest.raises(ValueError):
            opt.fold_l2(1e-4, m.named_parameters(), "l1")
        opt.fold_l2(1e-4, m.named_parameters(), "slimmable")
        assert opt._l2_ids == {id(m.weight)}
    with pytest.raises(NotImplementedError):
        l2_mask(m.named_parameters(), "mnas_no_bias")
    with pytest.raises(NotImplementedError):
        so.l2_decay_mask([], "mnas_no_bias")


def test_struct_size_and_no_device(built_lib):
    from yet_another_mobilenet_series_b200 import native
    assert built_lib.yamb_struct_size(24) == ctypes.sizeof(native.Sgd)
    assert built_lib.yamb_version() >= 101
    a = native.Sgd()
    a.n, a.p, a.g, a.mom = 64, 256, 512, 768
    a.lr, a.momentum, a.nesterov = 0.1, 0.9, 1
    bad = []
    for field, v in (("lr", -1.0), ("momentum", -1.0), ("dampening", -0.5),
                     ("weight_decay", -1.0)):
        b = native.Sgd.from_buffer_copy(a)
        b.nesterov = 0
        setattr(b, field, v)
        bad.append(b)
    b = native.Sgd.from_buffer_copy(a)
    b.momentum = 0.0                         # nesterov without momentum
    bad.append(b)
    b = native.Sgd.from_buffer_copy(a)
    b.dampening = 0.1                        # nesterov with dampening
    bad.append(b)
    b = native.Sgd.from_buffer_copy(a)
    b.mom = None                             # momentum without its arena
    bad.append(b)
    for b in bad:
        assert built_lib.yamb_sgd_step(ctypes.byref(b), None) == -1, built_lib.yamb_last_error()
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert built_lib.yamb_sgd_step(ctypes.byref(a), None) == -2
    assert b"no CUDA device" in built_lib.yamb_last_error()


CTOR_CASES = [dict(lr=-1), dict(momentum=-1), dict(weight_decay=-1),
              dict(nesterov=True), dict(nesterov=True, momentum=0.0),
              dict(nesterov=True, momentum=0.9, dampening=0.1), dict(lr=torch.tensor([0.1, 0.2])),
              dict(lr=0.1), dict(lr=0.1, momentum=0.9, dampening=0.5),
              dict(lr=0.1, momentum=0.9, nesterov=True, weight_decay=1e-4),
              dict(lr=0.1, dampening=-1.0), dict(lr=0.1, foreach=True), dict(lr=0.1, fused=True)]


@pytest.mark.parametrize("kw", CTOR_CASES, ids=[str(i) for i in range(len(CTOR_CASES))])
def test_ctor_errors_match_torch(kw):
    from yet_another_mobilenet_series_b200.fused_sgd import SGD

    def outcome(cls):
        try:
            cls([nn.Parameter(torch.zeros(3))], **kw)
        except ValueError as e:
            return "ValueError: %s" % e
        return "ok"

    assert outcome(SGD) == outcome(torch.optim.SGD)


def test_ctor_surface():
    from yet_another_mobilenet_series_b200 import native
    from yet_another_mobilenet_series_b200.fused_sgd import SGD
    p = [nn.Parameter(torch.zeros(3))]
    ours, theirs = SGD(p, lr=0.2, momentum=0.9, nesterov=True), torch.optim.SGD(
        p, lr=0.2, momentum=0.9, nesterov=True)
    assert ours.param_groups[0].keys() == theirs.param_groups[0].keys()
    assert {k: v for k, v in ours.defaults.items() if k not in ("foreach", "fused")} == \
        {k: v for k, v in theirs.defaults.items() if k not in ("foreach", "fused")}
    assert SGD(p).defaults["lr"] == torch.optim.SGD(p).defaults["lr"] == 1e-3
    for kw in (dict(maximize=True), dict(differentiable=True)):
        with pytest.raises(native.NativeError):
            SGD(p, lr=0.1, **kw)
    with pytest.raises(native.NativeError):     # no CPU fallback
        SGD(p, lr=0.1).step()
