"""The deferred layer reset's cases (test_gpu_layer_init.py: poisoned slabs, every writer against the eager reset) on
the emulated kernels (tests/emu), so that a cell a writer leaves unwritten is caught on a box without a GPU too."""
import os
import subprocess
import sys

from common import ROOT


def test_layer_init_cases_on_the_emulated_kernels():
    env = dict(os.environ, AMB_TEST_EMU="1")
    for k in ("AMB_EAGER_LAYER_INIT", "AMB_DSM_PRECISION", "AMB_DSM_STREAM_CHUNKS", "AMB_ORTHO_DOMINANCE",
              "AMB_COMPACT_MIRRORS", "AMB_EMU_SCHED"):
        env.pop(k, None)
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider",
           os.path.join(ROOT, "tests", "test_gpu_layer_init.py")]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    tail = "\n".join((r.stdout + r.stderr).splitlines()[-25:])
    assert r.returncode == 0, tail
    assert " passed" in tail and "failed" not in tail and "skipped" not in tail, tail
