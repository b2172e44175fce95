"""ORACLE tooling — the model kwargs of the AtomNAS zoo (every block of which, past the first, has
several depthwise branches) as the reference's own config loader resolves them, in the format of
oracle/make_model_cfgs.py (same child process).  Run in the build container only:

    python oracle/make_model_cfgs_multi_branch.py

Output: tests/golden/model_cfgs_multi_branch.json (travels to the GPU box; the reference does not).
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.make_model_cfgs import CHILD, REF, ROOT  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "model_cfgs_multi_branch.json")

CONFIGS = {
    "atomnas_a": "apps/searched/atomnas_a/atomnas_a.yml",
    "atomnas_b": "apps/searched/atomnas_b/atomnas_b.yml",
    "atomnas_c": "apps/searched/atomnas_c/atomnas_c.yml",
    "atomnas_a+": "apps/searched/atomnas_a/atomnas_a+.yml",
    "atomnas_b+": "apps/searched/atomnas_b/atomnas_b+.yml",
    "atomnas_c+": "apps/searched/atomnas_c/atomnas_c+.yml",
}


def main():
    env = dict(os.environ, ARNOLD_OUTPUT="/tmp/yamb_out", DATA_LMDB="/tmp/yamb_lmdb",
               PYTHONPATH=REF)
    res = {}
    for name, yml in CONFIGS.items():
        p = subprocess.run([sys.executable, "-c", CHILD, "app:" + os.path.join(REF, yml)],
                           cwd=REF, env=env, capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError("%s: %s" % (yml, p.stderr[-2000:]))
        line = [l for l in p.stdout.splitlines() if l.startswith("@@")][-1]
        res[name] = json.loads(line[2:])
        res[name]["yml"] = yml
        print(name, res[name]["n_params"], "params,", len(res[name]["state_shapes"]), "state keys")
    with open(OUT, "w") as f:
        json.dump(res, f, indent=0, sort_keys=True)


if __name__ == "__main__":
    main()
