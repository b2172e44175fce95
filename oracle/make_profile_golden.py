"""ORACLE tooling — what the LIVE reference's `utils.model_profiling.model_profiling` reports for
the networks of the reference's model zoo, built through the reference's own yml loader (as
oracle/make_model_cfgs.py does), plus the odd-width searched network of tests/test_searched_gpu.py.
Run in the build container only:

    python oracle/make_profile_golden.py

The profiler runs on CPU (`use_cuda=False`) with its `run_forward` stubbed to 0: the reference's
version calls `torch.cuda.synchronize()` even on CPU, and only the counts are wanted here.

Output: tests/golden/profile_rows.json.gz (gzip-compressed JSON), one entry per network:
  model, model_kwparams, image_size  what `Model(**model_kwparams, input_size=image_size)` takes
  header, total                      the table's header and separator lines, and its Total line
                                     (time 0; an AutoNL Total shows float MACs, from the
                                     non-local block's `nl_c`)
  rows                               the row names, in the order they were logged
  counts                             {module name: [n_macs, n_params]} of every module the
                                     profiler set them on ('' is the model)
`utils.config` parses sys.argv at import (utils/config.py:216), hence one subprocess per network.
"""
import gzip
import json
import os
import subprocess
import sys

REF = os.environ.get("YAMB_REFERENCE", "/root/reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "profile_rows.json.gz")

YMLS = {
    "mobilenet_v2": "apps/mobilenet/mobilenet_v2_mnas.yml",
    "proxyless_mobile": "apps/mobilenet/proxyless_mobile_mnas.yml",
    "single_path": "apps/mobilenet/single_path_nas_mnas.yml",
    "atomnas_a": "apps/searched/atomnas_a/atomnas_a.yml",
    "atomnas_b": "apps/searched/atomnas_b/atomnas_b.yml",
    "atomnas_c": "apps/searched/atomnas_c/atomnas_c.yml",
    "atomnas_a+": "apps/searched/atomnas_a/atomnas_a+.yml",
    "atomnas_b+": "apps/searched/atomnas_b/atomnas_b+.yml",
    "atomnas_c+": "apps/searched/atomnas_c/atomnas_c+.yml",
    "autonl_s": "apps/searched/autonl/autonl_s.yml",
    "autonl_l": "apps/searched/autonl/autonl_l.yml",
}

# tests/test_searched_gpu.py: several kernel sizes per block, SE, Swish, hidden widths 36 and 20
# (not multiples of 8), in both block packings, at 64x64
_ROWS = [[16, 1, 1, [3], [32], False],
         [24, 2, 2, [3, 5], [48, 24], True],
         [40, 2, 2, [3, 5, 7], [64, 36, 20], True],
         [80, 1, 2, [3], [160], True],
         [96, 1, 2, [3, 5], [96, 64], True]]
SEARCHED = {
    "searched_odd_fused": dict(
        inverted_residual_setting=_ROWS, block="InvertedResidualChannelsFused", se_ratio=0.5,
        active_fn="nn.Swish", batch_norm_momentum=0.01, batch_norm_epsilon=1e-3, num_classes=50,
        dropout_ratio=0.0, last_channel=320),
    "searched_odd_unfused": dict(
        inverted_residual_setting=_ROWS, block="InvertedResidualChannels", active_fn="nn.ReLU6",
        batch_norm_momentum=0.01, batch_norm_epsilon=1e-3, num_classes=50, dropout_ratio=0.0,
        last_channel=320),
}

CHILD = r"""
import importlib, json, logging, os
from utils.config import FLAGS
import utils.model_profiling as mp

def plain(v):
    if isinstance(v, dict):
        return {k: plain(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [plain(x) for x in v]
    return v

spec = os.environ.get("YAMB_PROFILE_SPEC")
if spec:
    spec = json.loads(spec)
else:
    spec = {"model": FLAGS.model, "model_kwparams": plain(dict(FLAGS.model_kwparams)),
            "image_size": FLAGS.image_size}
lines = []

class Keep(logging.Handler):
    def emit(self, record):
        msg = record.getMessage()
        if not msg.startswith("WARNING: leaf module"):
            lines.append(msg)

root = logging.getLogger()
root.handlers[:] = [Keep()]
root.setLevel(logging.INFO)
mp.run_forward = lambda self, input: 0
rows = []
row_of = mp.module_profiling

def module_profiling(self, input, output, verbose):
    n = len(lines)
    row_of(self, input, output, verbose)
    if len(lines) > n:
        rows.append(self.name)

mp.module_profiling = module_profiling
lib = importlib.import_module(spec["model"])
model = lib.Model(**spec["model_kwparams"], input_size=spec["image_size"])
size = spec["image_size"]
n_macs, n_params = mp.model_profiling(model, size, size, use_cuda=False, verbose=True)
counts = {name: [int(m.n_macs), int(m.n_params)] for name, m in model.named_modules()
          if hasattr(m, "n_macs")}
table = lines[next(i for i, l in enumerate(lines) if l.startswith("Item")):]
assert len(table) == len(rows) + 4
spec.update(header=table[:2], total=table[-1], rows=rows, counts=counts, n_macs=int(n_macs),
            n_params=int(n_params))
print("@@" + json.dumps(spec))
"""


def _run(env, yml):
    p = subprocess.run([sys.executable, "-c", CHILD, "app:" + os.path.join(REF, yml)],
                       cwd=REF, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError("%s: %s" % (yml, p.stderr[-2000:]))
    line = [l for l in p.stdout.splitlines() if l.startswith("@@")][-1]
    return json.loads(line[2:])


def main():
    env = dict(os.environ, ARNOLD_OUTPUT="/tmp/yamb_out", DATA_LMDB="/tmp/yamb_lmdb",
               PYTHONPATH=REF)
    res = {}
    for name, yml in YMLS.items():
        res[name] = _run(env, yml)
        res[name]["yml"] = yml
    for name, kw in SEARCHED.items():
        spec = {"model": "models.searched_network", "model_kwparams": kw, "image_size": 64}
        res[name] = _run(dict(env, YAMB_PROFILE_SPEC=json.dumps(spec)), YMLS["mobilenet_v2"])
    for name, r in res.items():
        print(name, "{:,} MACs, {:,} params, {} rows".format(r["n_macs"], r["n_params"],
                                                            len(r["rows"])))
    with gzip.GzipFile(OUT, "wb", mtime=0) as f:
        f.write(json.dumps(res, sort_keys=True, separators=(",", ":")).encode())


if __name__ == "__main__":
    main()
