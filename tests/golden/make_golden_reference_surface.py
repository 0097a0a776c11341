#!/usr/bin/env python
"""Generate tests/golden/reference_surface.json: the plugin surface of the reference that this package mirrors, read from the reference
sources once so that the tests compare against it without the reference tree.

    python tests/golden/make_golden_reference_surface.py [REFERENCE_ROOT]

For each of the five algorithms: every key of its default_config.py's get_config("x") with its value, and the parameter names of every
method of its model class (read from the source with ast, as the runner's duck typing sees them).
"""
import ast
import json
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

ALGORITHMS = {  # name: (default_config.py, model class source, model class name), relative to the reference root
    "ppo": ("rl_x/algorithms/ppo/pytorch/default_config.py", "rl_x/algorithms/ppo/pytorch/ppo.py", "PPO"),
    "sac": ("rl_x/algorithms/sac/pytorch/default_config.py", "rl_x/algorithms/sac/pytorch/sac.py", "SAC"),
    "fastsac": ("rl_x/algorithms/fastsac/pytorch/default_config.py", "rl_x/algorithms/fastsac/pytorch/fastsac.py", "FastSAC"),
    "espo": ("rl_x/algorithms/espo/pytorch/default_config.py", "rl_x/algorithms/espo/pytorch/espo.py", "ESPO"),
    "ppo_lstm": ("rl_x/algorithms/ppo_lstm/flax/default_config.py", "rl_x/algorithms/ppo_lstm/flax/ppo_lstm.py", "PPO_LSTM"),
}


def class_methods(path, cls):
    """{method name: [parameter names without cls]} of class `cls` in the source file `path`."""
    with open(path) as fh:
        tree = ast.parse(fh.read())
    for node in ast.walk(tree):
        if isinstance(node, ast.ClassDef) and node.name == cls:
            return {f.name: [a.arg for a in f.args.args if a.arg != "cls"] for f in node.body if isinstance(f, ast.FunctionDef)}
    raise AssertionError(f"no class {cls} in {path}")


def main(ref_root):
    from oracle import ref_arm
    ref_arm._install_stub()  # the reference's default configs import ml_collections
    out = {}
    for algo, (config_py, model_py, cls) in ALGORITHMS.items():
        cfg = runpy.run_path(os.path.join(ref_root, config_py))["get_config"]("x")
        out[algo] = {"config": {k: cfg[k] for k in cfg}, "class": cls, "methods": class_methods(os.path.join(ref_root, model_py), cls)}
    path = os.path.join(HERE, "reference_surface.json")
    with open(path, "w") as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print(path)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
