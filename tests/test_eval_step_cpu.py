"""CPU: the ABI of the eval-mode stem / head kernels, the CPU refusals of EvalStep / TrainStep, and
the reduction of per-rank validation sums to the reference's result keys (train.py:273-309)."""
import ctypes as C

import pytest
import torch

from yet_another_mobilenet_series_b200 import engine
from yet_another_mobilenet_series_b200 import native as nat
from yet_another_mobilenet_series_b200 import trainer


def test_new_structs_match_the_library(built_lib):
    assert built_lib.yamb_struct_size(25) == C.sizeof(nat.StemConvEval)
    assert built_lib.yamb_struct_size(26) == C.sizeof(nat.HeadPoolEval)
    assert nat.StemConvEval.conv.offset == 0
    assert C.sizeof(nat.StemConvEval) > C.sizeof(nat.StemConv)
    for name in ("yamb_stem_conv_eval_fwd", "yamb_head_pool_eval_fwd"):
        assert name in nat.SYMBOLS and hasattr(built_lib, name)


def test_tail_switch_is_off_by_default():
    assert engine.EVAL_TAIL_FUSED is False


def _tiny_model():
    from yet_another_mobilenet_series_b200 import mobilenet_supernet as sup
    rows = [[1, 16, 1, 1, [3]], [6, 24, 1, 2, [3]]]
    return sup.Model(num_classes=8, input_size=32, inverted_residual_setting=rows,
                     last_channel=64)


def test_eval_step_refuses_a_cpu_model():
    with pytest.raises(RuntimeError, match="CUDA"):
        trainer.EvalStep(_tiny_model(), 4, image_size=32)


def test_train_step_refuses_a_cpu_model():
    # ema_model() / validate() live on a TrainStep, which needs the model on CUDA
    with pytest.raises(RuntimeError, match="CUDA"):
        trainer.TrainStep(_tiny_model(), 4, image_size=32)


def test_metrics_from_per_rank_sums():
    g = torch.Generator().manual_seed(0)
    loss = torch.rand(3, 50, generator=g, dtype=torch.float64) * 5
    c1 = (torch.rand(3, 50, generator=g) < 0.6).long()
    c5 = torch.maximum(c1, (torch.rand(3, 50, generator=g) < 0.3).long())
    # what every rank accumulates, then the all-reduce SUM over the ranks
    per_rank = [(float(loss[r].sum()), int(c1[r].sum()), int(c5[r].sum()), 50) for r in range(3)]
    summed = [sum(col) for col in zip(*per_rank)]
    res = trainer.metrics_from_sums(*summed)
    assert set(res) == {"loss", "top1_error", "top5_error"}
    # the reference's meters: per-sample lists over every rank, averaged
    assert res["loss"] == pytest.approx(float(loss.mean()), rel=1e-12)
    assert res["top1_error"] == pytest.approx(float((1 - c1.double()).mean()), rel=1e-12)
    assert res["top5_error"] == pytest.approx(float((1 - c5.double()).mean()), rel=1e-12)
    with pytest.raises(ValueError):
        trainer.metrics_from_sums(0.0, 0, 0, 0)
