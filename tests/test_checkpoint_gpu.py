"""GPU: TrainStep checkpoints, resuming and partial last batches.

1. Resume is bit-exact: 6 uninterrupted steps (graph captured at step 3) against 3 steps,
   save_status, a NEW model of another init seed and a new TrainStep, load_state_dict, steps 4-6.
   Loss, parameters, optimizer state, EMA shadows, stat_shadow, running statistics and
   num_batches_tracked and the validate() metrics agree bit for bit at every step; RMSprop
   ('mnas') and Nesterov SGD ('slimmable') on a small MobileNetV2, RMSprop on AtomNAS-C+ and
   AutoNL-L (Squeeze-and-Excitation, non-local).
2. After the capture, `ts.load_state_dict(ts.state_dict())` keeps the graph object and
   `ts.opt.load_state_dict(...)` (new arenas) makes the step capture again; both continue run A's
   bits.
3. A partial batch (B, B, B, partial, B) runs eagerly between graph replays and matches the same
   sequence with use_graph=False bit for bit; bf16 and uint8 input.
4. The checkpoint has the key set, 'ema' layout, dtypes and shapes of one the reference's
   save_status wrote (tests/golden/ckpt_ref.pt, oracle/make_checkpoint.py), and that checkpoint
   loads into TrainStep.
Dropout is switched off where bits are compared: its stream differs between capture and eager."""
import importlib
import json
import os
import sys
import types

import pytest
import torch

from _cfg import MODULE_MAP, ROOT, load_cfgs

pytestmark = pytest.mark.gpu
B = 16
SIZE = {"mbv2": 64, "atomnas_c+": 128, "autonl_l": 128}
PARTIAL = B * 146 // 256          # the last batch of an 8-GPU ImageNet epoch, scaled to B
SGD = dict(optimizer="sgd", nesterov=True, weight_decay_method="slimmable", base_lr=0.1)
MEAN_STD = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


@pytest.fixture
def flags(monkeypatch):
    """A stand-in for the reference's utils.config (the non-local block reads FLAGS)."""
    mod = types.ModuleType("utils.config")
    mod.FLAGS = types.SimpleNamespace()
    monkeypatch.setitem(sys.modules, "utils.config", mod)
    return mod


def _model(kind, seed):
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb
    from yet_another_mobilenet_series_b200 import mobilenet_supernet as sup
    torch.manual_seed(seed)
    if kind == "mbv2":
        rows = [[1, 16, 1, 1, [3]], [6, 24, 2, 2, [3]], [6, 32, 1, 2, [5]], [6, 64, 1, 2, [3]],
                [6, 96, 1, 2, [3]]]
        model = sup.Model(num_classes=100, input_size=SIZE[kind], inverted_residual_setting=rows,
                          active_fn="nn.ReLU", batch_norm_momentum=0.01,
                          batch_norm_epsilon=1e-3, last_channel=128)
    else:
        cfg = load_cfgs()[kind]
        lib = importlib.import_module(MODULE_MAP[cfg["flags"]["model"]])
        model = lib.Model(**cfg["model_kwparams"], input_size=SIZE[kind])
    model.apply(mb.init_weights_mnas)
    for m in model.modules():
        if isinstance(m, mb.Nonlocal):
            m.bn.weight.data.fill_(0.5)        # ZeroInitBN would switch the non-local branch off
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return model.cuda()


def _batch(kind, i, n=B, u8=False):
    g = torch.Generator().manual_seed(100 + i)
    x = torch.randn(n, 3, SIZE[kind], SIZE[kind], generator=g)
    x = (x * 40 + 128).clamp(0, 255).to(torch.uint8) if u8 else x.to(torch.bfloat16)
    return x, torch.randint(0, 100, (n,), generator=g)


def _ts(kind, model, opt_kw, **kw):
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    return TrainStep(model, B, image_size=SIZE[kind], **opt_kw, **kw)


def _snap(ts, loss, val=None):
    """Everything a step leaves behind, cloned."""
    out = {"loss": loss.clone()}
    for n, p in ts.model.named_parameters():
        out["p." + n] = p.detach().clone()
        out["ema." + n] = ts.opt.ema_shadow(p).clone()
        for k, v in ts.opt.state.get(p, {}).items():
            out["opt.%s.%s" % (n, k)] = v.clone() if torch.is_tensor(v) else torch.tensor(v)
    for n, b in ts.model.named_buffers():
        out["buf." + n] = b.clone()
    for i, s in enumerate(ts.stat_shadow):
        out["stat_shadow.%d" % i] = s.clone()
    if val is not None:
        m = ts.validate([val])
        out.update({"val." + k: torch.tensor(v, dtype=torch.float64) for k, v in m.items()})
    return out


def _same(a, b):
    assert a.keys() == b.keys(), sorted(set(a) ^ set(b))[:5]
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, diff[:5]


def _steps(ts, kind, idx, val):
    return [_snap(ts, ts(*_batch(kind, i)), val) for i in idx]


def _run_a(kind, opt_kw, val):
    ts = _ts(kind, _model(kind, 0), opt_kw)
    snaps = _steps(ts, kind, range(6), val)
    assert ts.graph is not None
    return snaps


CASES = [("mbv2", "rmsprop"), ("mbv2", "sgd"), ("atomnas_c+", "rmsprop"), ("autonl_l", "rmsprop")]


@pytest.mark.parametrize("kind,opt", CASES)
def test_resume_is_bit_exact(built_lib, flags, tmp_path, kind, opt):
    opt_kw = SGD if opt == "sgd" else {}
    val = _batch(kind, 99)
    a = _run_a(kind, opt_kw, val)
    ts = _ts(kind, _model(kind, 0), opt_kw)
    for i, s in enumerate(_steps(ts, kind, range(3), val)):
        _same(a[i], s)
    assert ts.graph is not None
    path = str(tmp_path / "latest_checkpoint.pt")
    ts.save_status(path, 0, 0.5, ({"train": 1.0}, {"val": 2.0}))
    del ts
    ck = torch.load(path, map_location="cpu")
    assert ck["last_epoch"] == 0 and ck["best_val"] == 0.5 and ck["global_step"] == 3
    assert ck["meters"] == ({"train": 1.0}, {"val": 2.0})
    ts = _ts(kind, _model(kind, 1), opt_kw)                 # another init: all of it is loaded
    ts.load_state_dict(ck)
    assert ts.global_step == 3
    for i, s in zip(range(3, 6), _steps(ts, kind, range(3, 6), val)):
        _same(a[i], s)
    assert ts.graph is not None


def test_load_after_capture(built_lib, flags):
    kind, val = "mbv2", _batch("mbv2", 99)
    a = _run_a(kind, {}, val)
    # in place: the captured graph keeps replaying
    ts = _ts(kind, _model(kind, 0), {})
    _steps(ts, kind, range(3), val)
    g = ts.graph
    assert g is not None
    ts.load_state_dict(ts.state_dict())
    for i, s in zip(range(3, 6), _steps(ts, kind, range(3, 6), val)):
        _same(a[i], s)
    assert ts.graph is g
    # the optimizer's own load_state_dict builds new arenas: the step captures again
    ts = _ts(kind, _model(kind, 0), {})
    _steps(ts, kind, range(3), val)
    g = ts.graph
    ts.opt.load_state_dict(ts.opt.state_dict())
    for i, s in zip(range(3, 6), _steps(ts, kind, range(3, 6), val)):
        _same(a[i], s)
    assert ts.graph is not None and ts.graph is not g


@pytest.mark.parametrize("u8", [False, True], ids=["bf16", "uint8"])
def test_partial_batch(built_lib, u8):
    kind = "mbv2"
    kw = dict(input_dtype=torch.uint8, input_norm=MEAN_STD) if u8 else {}
    sizes = [B, B, B, PARTIAL, B]
    runs, graphs = [], []
    for use_graph in (True, False):
        ts = _ts(kind, _model(kind, 0), {}, use_graph=use_graph, **kw)
        snaps = []
        for i, n in enumerate(sizes):
            snaps.append(_snap(ts, ts(*_batch(kind, i, n, u8))))
            graphs.append(ts.graph)
        runs.append(snaps)
    for s, e in zip(*runs):
        _same(s, e)
    assert graphs[2] is not None and graphs[2] is graphs[3] is graphs[4]
    assert graphs[5:] == [None] * 5


def _golden():
    with open(os.path.join(ROOT, "tests", "golden", "ckpt_ref.json")) as f:
        meta = json.load(f)
    return meta, torch.load(os.path.join(ROOT, "tests", "golden", "ckpt_ref.pt"))


def _small_ts(meta):
    from yet_another_mobilenet_series_b200 import mobilenet_supernet as sup
    from yet_another_mobilenet_series_b200.trainer import TrainStep
    kw = dict(meta["net_kw"])
    torch.manual_seed(5)
    model = sup.Model(**kw).cuda()
    return TrainStep(model, meta["batch"], image_size=kw["input_size"])


def _layout(t):
    return (t.dtype, tuple(t.shape))


def test_layout_of_reference_checkpoint(built_lib, tmp_path):
    meta, ref = _golden()
    ts = _small_ts(meta)
    n = meta["batch"]
    for i in range(3):
        g = torch.Generator().manual_seed(i)
        ts(torch.randn(n, 3, 32, 32, generator=g).to(torch.bfloat16),
           torch.randint(0, 10, (n,), generator=g))
    path = str(tmp_path / "ckpt.pt")
    ts.save_status(path, 0, 0.5, None)
    ours = torch.load(path, map_location="cpu")
    assert set(ours) == set(ref) | {"global_step", "cuda_rng_state"}
    assert list(ours["model"]) == list(ref["model"])
    assert all(_layout(ours["model"][k]) == _layout(v) for k, v in ref["model"].items())
    oe, re_ = ours["ema"], ref["ema"]
    assert set(oe) == set(re_) and oe["param"] == re_["param"]
    assert list(oe["shadow"]) == list(re_["shadow"]) == list(oe["info"]) == list(re_["info"])
    assert all(_layout(oe["shadow"][k]) == _layout(v) for k, v in re_["shadow"].items())
    assert all(oe["info"][k] == v for k, v in re_["info"].items())   # 3 updates each
    oo, ro = ours["optimizer"], ref["optimizer"]
    assert oo["param_groups"][0].keys() == ro["param_groups"][0].keys()
    assert oo["state"].keys() == ro["state"].keys()
    for i, st in ro["state"].items():
        assert oo["state"][i].keys() == st.keys()
        assert all(_layout(oo["state"][i][k]) == _layout(v) for k, v in st.items()
                   if torch.is_tensor(v))


def test_load_reference_checkpoint(built_lib):
    meta, ref = _golden()
    ts = _small_ts(meta)
    ts.load_state_dict(ref)
    shadow, info = ref["ema"]["shadow"], ref["ema"]["info"]
    assert ts.global_step == next(iter(info.values()))["num_updates"] == meta["steps"]
    params = dict(ts.model.named_parameters())
    for k, v in ref["model"].items():
        assert torch.equal(ts.model.state_dict()[k[len("module."):]].cpu(), v), k
    for k, p in params.items():
        assert torch.equal(ts.opt.ema_shadow(p).cpu(), shadow[k]), k
    stat_names = [k for k in shadow if k not in params]
    assert all(torch.equal(s.cpu(), shadow[k]) for s, k in zip(ts.stat_shadow, stat_names))
    for i, p in enumerate(params.values()):
        for k, v in ref["optimizer"]["state"][i].items():
            got = ts.opt.state[p][k]
            assert (torch.equal(got.cpu(), v) if torch.is_tensor(v) else got == v), (i, k)
    n = meta["batch"]
    loss = ts(torch.randn(n, 3, 32, 32).to(torch.bfloat16), torch.randint(0, 10, (n,)))
    assert torch.isfinite(loss) and ts.global_step == meta["steps"] + 1
