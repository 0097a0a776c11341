#!/usr/bin/env python
"""Recipe that adds the reference's FastTD3 PyTorch modules to oracle/_ref, next to what oracle/make_ref.py stages there.

TEST INFRASTRUCTURE ONLY (nothing under rl_x_b200/ may import this or oracle/_ref).  The modules are copied byte for byte out of the reference
tree into the same git-ignored oracle/_ref/rl_x/... tree, so that `import rl_x.algorithms.fasttd3.pytorch.fasttd3` works once
oracle/ref_arm.import_reference() has put oracle/_ref on sys.path.  They are used by the checkpoint interop test of
tests/test_fasttd3_emulation.py (the reference's own FastTD3.save() / load()); nothing times them.  Run in the build container:

    python oracle/make_ref_fasttd3.py      # also called by __graft_entry__.build() when the reference tree is present

A manifest of their sha256 (oracle/_ref/MANIFEST_fasttd3.json) is written next to them so that a stale or edited copy is detectable.
"""
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
if os.path.dirname(HERE) not in sys.path:
    sys.path.insert(0, os.path.dirname(HERE))
from oracle import make_ref  # noqa: E402

DST = make_ref.DST
MANIFEST = os.path.join(DST, "MANIFEST_fasttd3.json")

FILES = [
    "rl_x/algorithms/fasttd3/__init__.py",
    "rl_x/algorithms/fasttd3/pytorch/__init__.py",
    "rl_x/algorithms/fasttd3/pytorch/critic.py",
    "rl_x/algorithms/fasttd3/pytorch/default_config.py",
    "rl_x/algorithms/fasttd3/pytorch/fasttd3.py",
    "rl_x/algorithms/fasttd3/pytorch/general_properties.py",
    "rl_x/algorithms/fasttd3/pytorch/observation_normalizer.py",
    "rl_x/algorithms/fasttd3/pytorch/policy.py",
    "rl_x/algorithms/fasttd3/pytorch/q_network.py",
    "rl_x/algorithms/fasttd3/pytorch/replay_buffer.py",
]


def available():
    """True when the base staging and these modules are present (here after build(), on the GPU box via the snapshot)."""
    return make_ref.available() and os.path.exists(MANIFEST)


def build_ref(ref_root=make_ref.REF_ROOT):
    """Stage the FastTD3 modules (after make_ref.build_ref()). Returns the destination, or None when the reference tree is absent."""
    if not os.path.isdir(os.path.join(ref_root, "rl_x")):
        return DST if available() else None
    manifest = {}
    for rel in FILES:
        src, dst = os.path.join(ref_root, rel), os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if not os.path.exists(src) and rel.endswith("__init__.py"):   # namespace-style package in the reference: an empty marker is enough
            open(dst, "a").close()
            manifest[rel] = "(empty package marker, absent in the reference)"
            continue
        shutil.copyfile(src, dst)
        manifest[rel] = make_ref._sha(dst)
    with open(MANIFEST, "w") as fh:
        json.dump({"source": ref_root, "files": manifest}, fh, indent=1, sort_keys=True)
    return DST


def verify():
    """sha256 of every staged FastTD3 file against its manifest."""
    with open(MANIFEST) as fh:
        man = json.load(fh)
    bad = [rel for rel, h in man["files"].items() if len(h) == 64 and make_ref._sha(os.path.join(DST, rel)) != h]
    if bad:
        raise RuntimeError(f"oracle/_ref's FastTD3 modules are not the staged reference any more: {bad}")
    return man


if __name__ == "__main__":
    make_ref.build_ref(sys.argv[1] if len(sys.argv) > 1 else make_ref.REF_ROOT)
    out = build_ref(sys.argv[1] if len(sys.argv) > 1 else make_ref.REF_ROOT)
    print(out or "reference tree not found; nothing staged")
