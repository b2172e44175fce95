"""CPU: the 'ema' entry of TrainStep's checkpoints has the layout of the reference's
ExponentialMovingAverage.state_dict() (utils/optim.py:87-95).

* Its variable names and their order equal those the reference's setup_ema (common.py:42-64)
  registers on its own MobileNetV2 and AtomNAS-C+ (fixture tests/golden/ckpt_ref.json, written
  by oracle/make_checkpoint.py).
* Built from name -> tensor maps by `trainer.ema_state_dict`, it loads into the live reference's
  ExponentialMovingAverage without a warning and comes back equal through its state_dict() (runs
  where the reference is installed; YAMB_REFERENCE names its directory)."""
import json
import os
import subprocess
import sys

import pytest
import torch

from _cfg import ROOT, build_from_cfg, load_cfgs

REF = os.environ.get("YAMB_REFERENCE", "/root/reference")
NAMES = ["mobilenet_v2", "atomnas_c+"]


def _golden():
    with open(os.path.join(ROOT, "tests", "golden", "ckpt_ref.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("name", NAMES)
def test_ema_names_match_reference_setup_ema(name):
    from yet_another_mobilenet_series_b200.trainer import ema_names
    model, _ = build_from_cfg(name)
    pnames, snames = ema_names(model)
    assert pnames + snames == _golden()["ema_names"][name]


def test_ema_state_dict_layout():
    from yet_another_mobilenet_series_b200.trainer import ema_state_dict
    shadow = {"a.weight": torch.ones(3), "a.running_mean": torch.zeros(2)}
    sd = ema_state_dict(shadow, 0, 0.99)
    assert list(sd) == ["info", "shadow", "param"]
    assert sd["param"] == {"momentum": 0.99, "zero_debias": False}
    assert list(sd["shadow"]) == list(shadow)
    assert all(sd["info"][n] == {"num_updates": 0, "last_momemtum": None, "zero_init": False}
               for n in shadow)
    sd = ema_state_dict(shadow, 5, 0.99)
    assert sd["info"]["a.weight"] == {"num_updates": 5, "last_momemtum": 6.0 / 15.0,
                                      "zero_init": False}
    assert ema_state_dict(shadow, 10 ** 6, 0.99)["info"]["a.weight"]["last_momemtum"] == 0.99


CHILD = r"""
import json, sys, warnings
from collections import OrderedDict
import torch
names, shapes, decay, base, gbatch = json.loads(sys.stdin.read())
from utils.optim import ExponentialMovingAverage
from yet_another_mobilenet_series_b200.trainer import ema_state_dict
g = torch.Generator().manual_seed(0)
shadow = OrderedDict((n, torch.randn(shapes[n], generator=g)) for n in names)
sd = ema_state_dict(shadow, 37, decay ** (gbatch / base))     # TrainStep's ema_decay
ema = ExponentialMovingAverage(ExponentialMovingAverage.adjust_momentum(decay, base / gbatch))
with warnings.catch_warnings():
    warnings.simplefilter("error")
    ema.load_state_dict(sd)
back = ema.state_dict()
assert list(back["shadow"]) == names and ema.average_names() == names
assert all(torch.equal(back["shadow"][n], shadow[n]) for n in names)
assert back["info"] == sd["info"] and back["param"] == sd["param"]
print("@@ok")
"""


@pytest.mark.parametrize("name", NAMES)
def test_ema_state_dict_loads_into_live_reference(name):
    if not os.path.isfile(os.path.join(REF, "utils", "optim.py")):
        pytest.skip("the reference is not installed here")
    cfg = load_cfgs()[name]
    names = _golden()["ema_names"][name]
    # the momentum setup_ema computes for 8 GPUs x per_gpu_batch_size must equal TrainStep's
    flags = cfg["flags"]
    args = [names, cfg["state_shapes"], flags["moving_average_decay"],
            flags["moving_average_decay_base_batch"], 8 * flags["per_gpu_batch_size"]]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([REF, ROOT]))
    p = subprocess.run([sys.executable, "-c", CHILD],
                       input=json.dumps(args),
                       env=env, cwd=ROOT, capture_output=True, text=True)
    assert p.returncode == 0 and "@@ok" in p.stdout, p.stderr[-3000:]
