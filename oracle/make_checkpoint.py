"""ORACLE tooling — a checkpoint written by the LIVE reference (/root/reference, imported
unmodified) for the checkpoint tests.  Run in the build container only:

    python oracle/make_checkpoint.py

Outputs (data only; they travel to the GPU box, /root/reference does not):
  tests/golden/ckpt_ref.pt     save_status (utils/common.py:122-133) of a 4-block network after
                               three reference training steps: DataParallel wrapper ('module.'
                               keys), RMSprop (utils/rmsprop.py), the EMA of setup_ema
                               (common.py:42-64) updated as train.py:103-114 does
  tests/golden/ckpt_ref.json   that network's kwargs and batch, and the EMA variable names in
                               setup_ema's registration order for MobileNetV2 and AtomNAS-C+

`utils.config` parses sys.argv at import (utils/config.py:216) and setup_ema reads FLAGS: one
child process per yml.
"""
import json
import os
import subprocess
import sys

REF = os.environ.get("YAMB_REFERENCE", "/root/reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")

NAME_CONFIGS = {"mobilenet_v2": "apps/mobilenet/mobilenet_v2_mnas.yml",
                "atomnas_c+": "apps/searched/atomnas_c/atomnas_c+.yml"}
# four single-block rows: the fewest blocks with which the Model's total stride reaches 32, which
# its classifier pooling assumes (AvgPool2d(input_size // 32))
NET_KW = dict(inverted_residual_setting=[[1, 8, 1, 2, [3]], [2, 8, 1, 2, [3]], [2, 16, 1, 2, [3]],
                                         [2, 16, 1, 2, [3]]],
              active_fn="nn.ReLU", batch_norm_momentum=0.01, batch_norm_epsilon=1e-3,
              input_size=32, num_classes=10, last_channel=64, dropout_ratio=0.0)
BATCH = 8
STEPS = 3


def child_names():
    """setup_ema's variable names on the model the yml describes."""
    import importlib
    import logging
    logging.disable(logging.CRITICAL)
    from utils.config import FLAGS
    import common as mc
    FLAGS.batch_size = FLAGS.per_gpu_batch_size
    lib = importlib.import_module(FLAGS.model)
    model = lib.Model(**FLAGS.model_kwparams, input_size=FLAGS.image_size)
    print("@@" + json.dumps(mc.setup_ema(model).average_names()))


def child_ckpt(path):
    """Three training steps of the reference's loop on a small network, then save_status."""
    import logging
    import warnings
    import torch
    logging.disable(logging.CRITICAL)
    warnings.simplefilter("ignore")
    from utils.config import FLAGS
    import common as mc
    import models.mobilenet_base as rmb
    import models.mobilenet_supernet as rsup
    from utils import optim as roptim
    from utils.common import save_status, get_params_by_name
    from utils.rmsprop import RMSprop
    FLAGS.batch_size = BATCH
    FLAGS.moving_average_decay = 0.9999
    FLAGS.moving_average_decay_adjust = True
    FLAGS.moving_average_decay_base_batch = 4096
    torch.manual_seed(1995)
    model = rsup.Model(**NET_KW)
    model.apply(rmb.init_weights_mnas)
    wrapper = torch.nn.DataParallel(model)
    opt = RMSprop(wrapper.parameters(), lr=0.016 * BATCH / 256, alpha=0.9, momentum=0.9, eps=1e-3,
                  eps_inside_sqrt=True, weight_decay=0)
    ema = mc.setup_ema(model)
    crit = roptim.CrossEntropyLabelSmooth(NET_KW["num_classes"], 0.1)
    g = torch.Generator().manual_seed(0)
    for step in range(1, STEPS + 1):
        x = torch.randn(BATCH, 3, 32, 32, generator=g)
        t = torch.randint(0, NET_KW["num_classes"], (BATCH,), generator=g)
        wrapper.train()
        opt.zero_grad()
        loss = crit(wrapper(x), t).mean() + roptim.cal_l2_loss(model, 1e-5, "mnas")
        loss.backward()
        opt.step()
        names = ema.average_names()
        for name, param in zip(names, get_params_by_name(model, names)):
            ema(name, param, step)
    save_status(wrapper, opt, ema, 0, 0.5, None, path)


def _run_child(mode, yml):
    """`mode`: 'names', or the path of the checkpoint to write.  The child's argv is the
    reference's (its config parser rejects anything else), so the mode travels in the
    environment."""
    env = dict(os.environ, ARNOLD_OUTPUT="/tmp/yamb_out", DATA_LMDB="/tmp/yamb_lmdb",
               PYTHONPATH=REF, YAMB_CKPT_CHILD=mode)
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "app:" + os.path.join(REF, yml)],
                       cwd=REF, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError("%s: %s" % (yml, p.stderr[-2000:]))
    return p.stdout


def main():
    names = {}
    for key, yml in NAME_CONFIGS.items():
        out = _run_child("names", yml)
        names[key] = json.loads([l for l in out.splitlines() if l.startswith("@@")][-1][2:])
        print(key, len(names[key]), "EMA variables")
    path = os.path.join(OUT, "ckpt_ref.pt")
    _run_child(path, NAME_CONFIGS["mobilenet_v2"])
    print("ckpt_ref.pt", os.path.getsize(path), "bytes")
    with open(os.path.join(OUT, "ckpt_ref.json"), "w") as f:
        json.dump({"net_kw": NET_KW, "batch": BATCH, "steps": STEPS, "ema_names": names}, f,
                  indent=0)


if __name__ == "__main__":
    mode = os.environ.get("YAMB_CKPT_CHILD")
    if mode == "names":
        child_names()
    elif mode:
        child_ckpt(mode)
    else:
        main()
