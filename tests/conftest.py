import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100: pytest -m gpu)")


def pytest_sessionfinish(session, exitstatus):
    """RLX_AUX_ENGINE_REPORT=<file>: leave "<tensor GEMMs> <persistent recurrence launches>" of this process - the FastSAC / PPO+LSTM GEMMs
    that ran on the wgmma engine and the one-launch-per-direction LSTM recurrences (the subprocess runs of run_suite_with_switches below read
    it back: a green suite that never took the path it was asked to take proves nothing)."""
    path = os.environ.get("RLX_AUX_ENGINE_REPORT")
    if path:
        try:
            from rl_x_b200 import _native as nt
            lib = nt.load()
            text = f"{int(lib.rlx_aux_tc_gemm_count())} {int(lib.rlx_lstm_persistent_launch_count())}"
        except Exception as exc:  # noqa: BLE001 - the report is best effort, the exit status carries the verdict
            text = f"unavailable: {exc}"
        with open(path, "w") as fh:
            fh.write(text)


def run_suite_with_switches(test_file, tmp_path, tensor_engine=False, persistent=False, timeout=900):
    """Run the GPU parity tests of `test_file` again in a SUBPROCESS with the opt-in paths on: RLX_AUX_GEMM_ENGINE=1 (dense layers on the wgmma
    3xTF32 engine where it covers the product) and / or RLX_LSTM_PERSISTENT=1 (LSTM recurrence as one block-cooperative launch per direction).
    A subprocess because a kernel that traps or faults takes the CUDA context with it: here that costs one test, not the rest of the
    session.  Returns (returncode, output tail, tensor GEMM count, persistent launch count); the counts are -1 when no report came back."""
    import subprocess
    report = os.path.join(str(tmp_path), "aux_paths.txt")
    env = dict(os.environ, RLX_AUX_GEMM_ENGINE="1" if tensor_engine else "0", RLX_LSTM_PERSISTENT="1" if persistent else "0", RLX_AUX_ENGINE_REPORT=report)
    proc = subprocess.run([sys.executable, "-m", "pytest", test_file, "-x", "-q", "-m", "gpu", "-k", "not subprocess", "-p", "no:cacheprovider"],
                          env=env, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    counts = open(report).read().split() if os.path.exists(report) else []
    tc, pers = (int(counts[0]), int(counts[1])) if len(counts) == 2 and all(x.isdigit() for x in counts) else (-1, -1)
    return proc.returncode, (proc.stdout + proc.stderr)[-3000:], tc, pers


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


class Golden:
    """Golden vectors captured from the executed reference (tests/golden/make_golden_ppo.py)."""

    def __init__(self, tag):
        self.z = np.load(os.path.join(GOLDEN_DIR, f"ppo_{tag}.npz"))
        m = self.z["meta"]
        self.N, self.T, self.obs, self.act, self.hidden, self.mb, self.epochs, self.iterations, self.seed = (int(x) for x in m)
        f = self.z["meta_f"]
        (self.gamma, self.gae_lambda, self.clip_range, self.entropy_coef, self.critic_coef, self.max_grad_norm, self.lr,
         self.std_dev, self.act_low, self.act_high) = (float(x) for x in f[:10])
        self.anneal = bool(f[10])
        self.B = self.N * self.T

    def __getitem__(self, k):
        return self.z[k]

    def params(self, prefix):
        """(policy dict, critic dict) of numpy arrays under e.g. 'init' or 'iter0'."""
        pol = {k.split("/", 2)[2]: self.z[k] for k in self.z.files if k.startswith(f"{prefix}/policy/")}
        cri = {k.split("/", 2)[2]: self.z[k] for k in self.z.files if k.startswith(f"{prefix}/critic/")}
        return pol, cri

    def perms(self, iteration):
        return [self.z[f"perm/{iteration * self.epochs + e}"] for e in range(self.epochs)]

    def lr_at(self, iteration):
        # LinearLR(start 1 -> end 0 over total_iters = iterations), stepped once per iteration (ppo.py:87-88,302-304)
        if not self.anneal:
            return self.lr
        return self.lr * (1.0 - iteration / self.iterations)


class GoldenEspo(Golden):
    """Golden vectors of the executed ESPO reference (tests/golden/make_golden_espo.py); same layout as the PPO files except that
    `epochs` is max_epochs, the third float is max_ratio_delta and the index arrays are `choice/<k>`."""

    def __init__(self, tag):
        self.z = np.load(os.path.join(GOLDEN_DIR, f"espo_{tag}.npz"))
        m = self.z["meta"]
        self.N, self.T, self.obs, self.act, self.hidden, self.mb, self.max_epochs, self.iterations, self.seed = (int(x) for x in m)
        self.epochs = self.max_epochs
        f = self.z["meta_f"]
        (self.gamma, self.gae_lambda, self.max_ratio_delta, self.entropy_coef, self.critic_coef, self.max_grad_norm, self.lr,
         self.std_dev, self.act_low, self.act_high) = (float(x) for x in f[:10])
        self.clip_range = float("inf")
        self.anneal = bool(f[10])
        self.B = self.N * self.T


@pytest.fixture(scope="session")
def golden_espo():
    return GoldenEspo("small")


@pytest.fixture(scope="session", params=["small", "humanoid"])
def golden(request):
    return Golden(request.param)


@pytest.fixture(scope="session")
def golden_small():
    return Golden("small")


@pytest.fixture(scope="session")
def golden_humanoid():
    return Golden("humanoid")


def emu_build_cmd(out, src):
    """g++ command of the host-emulation builds (tests/test_*_emulation.py).  RLX_EMU_CXXFLAGS adds flags, e.g. an AddressSanitizer pass
    over the emulated kernels:  RLX_EMU_CXXFLAGS="-g -fsanitize=address" LD_PRELOAD=$(gcc -print-file-name=libasan.so)
    ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_lstm_emulation.py tests/test_fastsac_emulation.py"""
    import os
    import shlex
    return (["g++", "-x", "c++", "-std=c++17", "-O1", "-fPIC", "-shared", "-pthread", "-DRLX_EMU"] + shlex.split(os.environ.get("RLX_EMU_CXXFLAGS", ""))
            + ["-o", str(out), str(src)])
