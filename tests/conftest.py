import os
import subprocess
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA GPU (run on an H100 with `pytest -m gpu`)")


def run_parallel(script, np=2, args=(), timeout=180, env=None, expect_fail=False, launcher_args=()):
    """Runs tests/parallel/<script> under `hvdrun -np <np>` on this host and returns (rc, output)."""
    e = os.environ.copy()
    e["PYTHONPATH"] = REPO + os.pathsep + e.get("PYTHONPATH", "")
    e.setdefault("HOROVOD_LOG_LEVEL", "warning")
    e.setdefault("OMP_NUM_THREADS", "1")
    if env:
        e.update(env)
    path = script if os.path.isabs(script) else os.path.join(REPO, "tests", "parallel", script)
    cmd = [sys.executable, "-m", "horovod_b200.runner.launch", "-np", str(np), *launcher_args, sys.executable, path, *args]
    # the timeout only guards against hangs: on a loaded or freshly started box (first `import torch` can take a minute per
    # process) a tight limit turns slowness into a failure, so never go below five minutes
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, env=e, timeout=max(timeout, 300), cwd=REPO)
    out = p.stdout.decode(errors="replace")
    if not expect_fail and p.returncode != 0:
        raise AssertionError(f"parallel run failed (rc={p.returncode}):\n{out[-6000:]}")
    return p.returncode, out


@pytest.fixture(scope="session")
def native_built():
    from horovod_b200 import build
    build.build_all()
    return True
