"""model_profiling without a device: the counts, row names and table of the reference's profiler
(tests/golden/profile_rows.json.gz, written by oracle/make_profile_golden.py from the live
reference on the networks of its model zoo) for this package's builders given the same keywords."""
import gzip
import importlib
import json
import logging
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODULE_MAP = {"models.mobilenet_supernet": "yet_another_mobilenet_series_b200.mobilenet_supernet",
              "models.searched_network": "yet_another_mobilenet_series_b200.searched_network"}

with gzip.open(os.path.join(ROOT, "tests", "golden", "profile_rows.json.gz"), "rt") as f:
    GOLDEN = json.load(f)


def build(name):
    g = GOLDEN[name]
    lib = importlib.import_module(MODULE_MAP[g["model"]])
    return lib.Model(**g["model_kwparams"], input_size=g["image_size"])


def profile(model, size, caplog, **kw):
    from yet_another_mobilenet_series_b200.model_profiling import model_profiling
    caplog.clear()
    with caplog.at_level(logging.INFO):
        result = model_profiling(model, size, size, **kw)
    return result, [r.getMessage() for r in caplog.records]


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_counts_rows_and_table_match_reference(name, caplog, monkeypatch):
    g = GOLDEN[name]
    model = build(name).train()

    def no_forward(*args):
        raise AssertionError("use_cuda=False must not run the network")
    monkeypatch.setattr(model, "forward", no_forward)
    (n_macs, n_params), lines = profile(model, g["image_size"], caplog, use_cuda=False)
    assert (n_macs, n_params) == (g["n_macs"], g["n_params"])
    counts = {k: [m.n_macs, m.n_params] for k, m in model.named_modules() if hasattr(m, "n_macs")}
    assert counts == g["counts"]
    assert not model.training
    # one line on the missing CPU timing, then the reference's table: its header and separator,
    # the rows in its order, each named as it names it and with that module's counts, the
    # separator and its Total line
    assert len(lines) == len(g["rows"]) + 5
    assert "no CPU timing" in lines[0]
    assert lines[1:3] == g["header"] and lines[-2] == g["header"][1]
    assert lines[-1] == g["total"]
    by_name = {}
    for m in model.modules():
        if hasattr(m, "name"):
            by_name.setdefault(m.name, set()).add(("{:,}".format(m.n_params),
                                                   "{:,}".format(m.n_macs)))
    assert sorted(by_name) == sorted(set(g["rows"]))
    for line, name in zip(lines[3:-2], g["rows"]):
        assert line.startswith(name)
        params, macs, secs = line[len(name):].split()
        assert (params, macs) in by_name[name] and secs == "0"
        assert line == name.ljust(95) + params.rjust(15) + macs.rjust(15) + secs.rjust(15)


def test_mobilenet_v2_totals(caplog):
    (n_macs, n_params), lines = profile(build("mobilenet_v2"), 224, caplog, use_cuda=False)
    assert (n_macs, n_params) == (300_836_992, 3_470_760)
    assert lines[-1] == "Total" + " " * 90 + "      3,470,760    300,836,992              0"


def test_batch_scales_macs_only(caplog):
    g = GOLDEN["mobilenet_v2"]
    model = build("mobilenet_v2")
    (n_macs, n_params), _ = profile(model, 224, caplog, batch=4, use_cuda=False, verbose=False)
    assert (n_macs, n_params) == (4 * g["n_macs"], g["n_params"])
    assert all(getattr(m, "n_seconds", 0) == 0 for m in model.modules())


def test_counts_the_user_visible_widths(caplog):
    """AtomNAS-style widths that are not multiples of 8 count as built (the kernels run a
    channel-padded copy): the depthwise row of a 20-channel branch holds 20 * 7 * 7 weights."""
    model = build("searched_odd_fused")
    profile(model, 64, caplog, use_cuda=False, verbose=False)
    dw = model.features[4].depth_ops[2][1][0]
    assert (dw.in_channels, dw.kernel_size) == (20, (7, 7))
    assert dw.n_params == 20 * 7 * 7
    assert dw.n_macs == 20 * 7 * 7 * 8 * 8


def test_unknown_container_raises(caplog):
    from yet_another_mobilenet_series_b200.model_profiling import model_profiling

    class Two(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.a, self.b = torch.nn.Conv2d(3, 8, 3), torch.nn.Conv2d(8, 8, 3)

    with pytest.raises(NotImplementedError, match="Two"):
        model_profiling(Two(), 32, 32, use_cuda=False, verbose=False)
