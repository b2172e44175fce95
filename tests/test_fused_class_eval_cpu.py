"""engine.eval_supported on InvertedResidualChannelsFused (AutoNL, AtomNAS): the eval-path rule of
that class.  It decides from module structure only, so no GPU is needed."""
import torch

from yet_another_mobilenet_series_b200 import engine
from yet_another_mobilenet_series_b200 import mobilenet_base as mb

BN = {"momentum": 0.01, "eps": 1e-3}
SWISH, RELU6 = mb.get_active_fn("nn.Swish"), mb.get_active_fn("nn.ReLU6")


def fused(inp, oup, stride, channels, ks, expand=True, act=SWISH, **kw):
    return mb.InvertedResidualChannelsFused(inp, oup, stride, channels, ks, expand, active_fn=act,
                                            batch_norm_kwargs=BN, **kw).eval()


def test_fused_class_eval_dispatch_rule(monkeypatch):
    monkeypatch.setattr(engine, "FUSED_CLASS_SHAPE_RULE", False)   # every shape the kernel covers
    x = torch.zeros(2, 80, 14, 14)
    se_nl = fused(80, 80, 1, [240], [3], se_ratio=0.25, nl_c=0.125, nl_s=2)
    assert not engine.eval_supported(se_nl, x)          # gradient mode is on
    with torch.no_grad():
        # accepted: SE, non-local, both, Swish k = 5 / 7 (stride 1 and 2), no expansion with k = 3
        assert engine.eval_supported(se_nl, x)
        assert engine.eval_supported(fused(80, 80, 1, [240], [3], se_ratio=0.25), x)
        assert engine.eval_supported(fused(80, 80, 1, [240], [3], nl_c=0.25, nl_s=1), x)
        assert engine.eval_supported(fused(80, 96, 1, [480], [5]), x)
        assert engine.eval_supported(fused(80, 96, 2, [480], [5], se_ratio=0.25), x)
        assert engine.eval_supported(fused(80, 80, 1, [240], [7], act=RELU6), x)
        assert engine.eval_supported(fused(192, 320, 1, [1152], [5], se_ratio=0.25,
                                           nl_c=0.25, nl_s=1), x)
        assert engine.eval_supported(fused(32, 16, 1, [32], [3], False, se_ratio=0.25), x)
        # rejected: several branches, odd widths, no expansion with k = 5, widths past the tiles
        assert not engine.eval_supported(fused(40, 40, 1, [40, 23, 28], [3, 5, 7]), x)
        assert not engine.eval_supported(fused(40, 40, 1, [120, 120], [3, 5]), x)
        assert not engine.eval_supported(fused(40, 40, 1, [90], [3]), x)
        assert not engine.eval_supported(fused(32, 16, 1, [32], [5], False), x)
        assert not engine.eval_supported(fused(264, 264, 1, [528], [3]), x)
        assert not engine.eval_supported(fused(192, 328, 1, [1152], [3]), x)
        # rejected: a BatchNorm in train mode (the non-local block's too), a non-BatchNorm nl_norm
        assert not engine.eval_supported(se_nl.train(), x)
        se_nl.eval()
        se_nl.nl_op.bn.train()
        assert not engine.eval_supported(se_nl, x)
        se_nl.eval()
        gn = fused(80, 80, 1, [240], [3], nl_c=0.25, nl_s=1)
        gn.nl_op.bn = torch.nn.GroupNorm(8, 80)
        assert not engine.eval_supported(gn, x)
        # the unfused class takes the path by its own rule; YAMB_EVAL_FUSED=0 turns it off
        plain = mb.InvertedResidualChannels(80, 80, 1, [240], [3], True, active_fn=RELU6,
                                            batch_norm_kwargs=BN).eval()
        assert engine.eval_supported(plain, x)
        prev, engine.EVAL_FUSED = engine.EVAL_FUSED, False
        try:
            assert not engine.eval_supported(se_nl, x)
        finally:
            engine.EVAL_FUSED = prev


def test_shape_rule():
    """The measured shape rule keeps 5x5 / 7x7 blocks and blocks without the expansion on the
    four-launch sequence."""
    x = torch.zeros(2, 80, 14, 14)
    with torch.no_grad():
        assert engine.FUSED_CLASS_SHAPE_RULE
        assert engine.eval_supported(fused(80, 80, 1, [240], [3], se_ratio=0.25), x)
        assert not engine.eval_supported(fused(80, 96, 1, [480], [5]), x)
        assert not engine.eval_supported(fused(80, 80, 1, [240], [7]), x)
        assert not engine.eval_supported(fused(32, 16, 1, [32], [3], False, se_ratio=0.25), x)


def test_autonl_and_atomnas_coverage(monkeypatch):
    """Every AutoNL-L block and AtomNAS-C+ block 1 (the single-branch one) are covered by the
    kernel; with the shape rule, the 3x3 AutoNL-L blocks with the expansion take the path."""
    from _cfg import build_from_cfg
    with torch.no_grad():
        for name, want, want_rule in (("autonl_l", 21, [3, 5, 6, 7, 9, 10, 11, 15]),
                                      ("atomnas_c+", 1, [])):
            model, _ = build_from_cfg(name)
            model.eval()
            blocks = [m for m in model.features if hasattr(m, "expand_conv")]
            x = torch.zeros(1, 8, 14, 14)
            got = [i for i, b in enumerate(blocks) if engine.eval_supported(b, x)]
            assert got == want_rule, (name, got)
            monkeypatch.setattr(engine, "FUSED_CLASS_SHAPE_RULE", False)
            got = [i for i, b in enumerate(blocks) if engine.eval_supported(b, x)]
            monkeypatch.setattr(engine, "FUSED_CLASS_SHAPE_RULE", True)
            assert len(got) == want, (name, got)
            if name == "atomnas_c+":
                assert got == [0]
