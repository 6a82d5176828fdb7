"""scikit-learn is needed by LC2ST only: without it, `sbi_b200.diagnostics` still imports and SBC / TARP still run,
and the LC2ST names raise an ImportError that names scikit-learn.  Checked in a fresh interpreter in which every
`sklearn` import fails."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCRIPT = r'''
import sys
sys.modules["sklearn"] = None          # `import sklearn` (and every sklearn.*) now raises ModuleNotFoundError
import torch
import sbi_b200.diagnostics as D


class Posterior:
    def sample_batched(self, shape, x, show_progress_bars=False):
        return torch.randn(shape[0], x.shape[0], 2)


theta = torch.randn(100, 2)
ranks, dap = D.run_sbc(theta, theta + 0.1, Posterior(), num_posterior_samples=100)
assert ranks.shape == (100, 2) and dap.shape == (100, 2)
ecp, alpha = D.run_tarp(theta, theta + 0.1, Posterior(), num_posterior_samples=100)
assert ecp.shape == alpha.shape
for name in ("LC2ST", "LC2ST_NF", "LC2STScores", "LC2STState"):
    try:
        getattr(D, name)
    except ImportError as e:
        assert "scikit-learn" in str(e), e
    else:
        raise AssertionError(name + " imported without scikit-learn")
try:
    from sbi_b200.diagnostics import LC2ST  # noqa: F401
except ImportError as e:
    assert "scikit-learn" in str(e), e
else:
    raise AssertionError("LC2ST imported without scikit-learn")
print("ok")
'''


def test_diagnostics_without_sklearn():
    r = subprocess.run([sys.executable, "-c", _SCRIPT], cwd=ROOT, capture_output=True, text=True,
                       env={**os.environ, "PYTHONPATH": ROOT + os.pathsep + os.environ.get("PYTHONPATH", "")})
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
