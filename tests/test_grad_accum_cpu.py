"""CPU: the arguments of TrainStep's gradient accumulation (`micro_batch`) and what a step derives
from them (trainer.step_hyper): the learning rate and the EMA decay follow the global batch
per_gpu_batch x world, and the optimizer's grad_scale = 1 / (world x k) turns the sum of k
micro-batch mean-loss gradients on every rank into the mean over the global batch."""
import math

import pytest
import torch

from yet_another_mobilenet_series_b200 import distributed as udist
from yet_another_mobilenet_series_b200 import trainer
from yet_another_mobilenet_series_b200.trainer import TrainStep, step_hyper


@pytest.mark.parametrize("micro", [0, -4, 3, 5, 32])
def test_micro_batch_must_divide_per_gpu_batch(micro):
    with pytest.raises(ValueError):
        step_hyper(16, micro, 1)
    # rejected before the model is looked at: a CPU model is not the error raised
    with pytest.raises(ValueError):
        TrainStep(torch.nn.Linear(4, 4), 16, micro_batch=micro)


def test_cpu_model_still_refused_with_a_valid_micro_batch():
    with pytest.raises(RuntimeError):
        TrainStep(torch.nn.Linear(4, 4), 16, micro_batch=4)


@pytest.mark.parametrize("per_gpu,micro,world", [
    (256, None, 1), (256, 256, 1), (512, 256, 1), (1024, 256, 1), (1024, 128, 1),
    (512, 128, 8), (4096, 128, 1), (128, 32, 32), (16, 4, 2)])
def test_derived_hyper_parameters(per_gpu, micro, world):
    mb, k, lr, decay, scale = step_hyper(per_gpu, micro, world, base_lr=0.016,
                                         base_total_batch=256, ema_decay=0.9999,
                                         ema_base_batch=4096)
    gbatch = per_gpu * world
    assert mb == (per_gpu if micro is None else micro)
    assert k == per_gpu // mb and k * mb == per_gpu
    # reference common.py:204-205 and :47-57, on the global batch of one optimizer step
    assert lr == 0.016 * gbatch / 256
    assert decay == 0.9999 ** (gbatch / 4096)
    assert math.isclose(scale * world * k, 1.0, rel_tol=1e-15)
    if k == 1:                         # the value TrainStep set before micro-batches existed
        assert scale == 1.0 / world


def test_recipe_batch_on_fewer_gpus_keeps_lr_and_decay():
    """The MnasNet recipe (128 images x 32 GPUs = 4096) reproduced on 8 GPUs and on 1 GPU derives
    the same learning rate and EMA decay; only the micro-batch count differs."""
    ref = step_hyper(128, None, 32)
    for per_gpu, world in ((512, 8), (4096, 1)):
        mb, k, lr, decay, scale = step_hyper(per_gpu, 128, world)
        assert (mb, lr, decay) == (128, ref[2], ref[3])
        assert k == 4096 // (128 * world) and scale == 1.0 / (world * k)
    assert ref[2] == 0.016 * 4096 / 256


def test_no_ema_without_decay():
    assert step_hyper(64, 16, 1, ema_decay=0)[3] is None


def test_world_size_reaches_the_derivation(monkeypatch):
    seen = {}
    real = trainer.step_hyper

    def spy(per_gpu, micro, world, *a):
        seen["world"] = world
        return real(per_gpu, micro, world, *a)

    monkeypatch.setattr(udist, "get_world_size_fallback", lambda: 4)
    monkeypatch.setattr(trainer, "step_hyper", spy)
    with pytest.raises(RuntimeError):              # CPU model: refused after the derivation
        TrainStep(torch.nn.Linear(4, 4), 64, micro_batch=16)
    assert seen["world"] == 4
