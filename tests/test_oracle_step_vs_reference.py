"""CPU: pin oracle/torch_model.py (the CPU-baseline port of the whole training step) against three
training steps of the reference classes, recorded in tests/golden/step.pt
(oracle/make_golden.py --step): the loss of every step, the final state and the EMA shadows."""
import os
import warnings

import torch

from oracle.make_golden import STEP_BATCH, STEP_KW


def test_port_step_equals_reference_step(golden_dir):
    warnings.simplefilter("ignore")
    from yet_another_mobilenet_series_b200 import mobilenet_base as mb, mobilenet_supernet as sup
    from oracle import torch_model as tm

    rec = torch.load(os.path.join(golden_dir, "step.pt"), weights_only=False)
    torch.manual_seed(1995)
    ours = sup.Model(**STEP_KW)
    ours.apply(mb.init_weights_mnas)
    port = tm.as_reference(ours)
    for m in port.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    B = STEP_BATCH
    trainer = tm.RefTrainer(port, B)
    g = torch.Generator().manual_seed(0)
    for step in range(1, 4):
        x = torch.randn(B, 3, 64, 64, generator=g)
        t = torch.randint(0, 10, (B,), generator=g)
        lp = trainer.step(x, t)
        loss = rec["losses"][step - 1]
        assert abs(lp - loss) < 1e-5 * max(1.0, abs(loss))
    sa, sb = rec["state"], port.state_dict()
    assert set(sa) == set(sb)
    for k in sa:
        assert torch.allclose(sa[k].float(), sb[k].float(), rtol=1e-5, atol=1e-6), k
    assert set(rec["ema"]) == set(trainer.ema.shadow)
    for n, v in rec["ema"].items():
        assert torch.allclose(v, trainer.ema.shadow[n], rtol=1e-5, atol=1e-6), n
