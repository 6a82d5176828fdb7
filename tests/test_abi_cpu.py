"""CPU checks of the boundary: the library builds for sm_90a, loads, and exports every symbol
include/sbi_b200.h declares; argument errors surface as the documented codes; the product path
refuses to run without a CUDA device (no CPU fallback)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_exported(lib):
    from sbi_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "sbi_b200.h")).read()
    declared = set(re.findall(r"\b(?:int64_t|int|void\*|void)\s+(sbi_b200_\w+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.exported_symbols())
    for name in declared:
        assert getattr(lib, name) is not None
    assert lib.sbi_b200_abi_version() == 1


def test_sass_has_tma_bulk_copy(lib):
    """The weight pipeline must be the TMA bulk-copy path (UBLKCP) for sm_90a, and the tensor-core
    kernels must run on warpgroup MMAs (HGMMA)."""
    import shutil
    import subprocess
    from sbi_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert "UBLKCP" in out
    assert "HGMMA" in out


def test_argument_errors(lib):
    from sbi_b200 import _lib as L
    assert lib.sbi_b200_reduce_partials(None, 1, 4, None, None) == -1
    assert lib.sbi_b200_adam_clip_step(None, None, None, None, None, 4, 1e-3, .9, .999, 1e-8, 5., 1., None) == -1
    # null pointers are refused before any CUDA call; the length and count checks behind them need device
    # pointers (tests/test_optim_gpu.py)
    assert lib.sbi_b200_reduce_partials_norm(None, 1, 4, None, None, None, None) == -1
    assert lib.sbi_b200_adam_clip_step_norm(None, None, None, None, None, 4, 1e-3, .9, .999, 1e-8, 5., 1., None, 0,
                                            None) == -1
    assert lib.sbi_b200_nll_stats(None, 4, None, None) == -1
    assert lib.sbi_b200_nll_stats(None, -1, None, None) == -1
    assert lib.sbi_b200_nsf_logprob(None, None, None, None, None) == -1
    with pytest.raises(ValueError):
        L.check(-1, "x")


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback():
    from oracle import sbi_port
    from sbi_b200.inference import NPE
    from sbi_b200.neural_nets import build_nsf
    theta, x = sbi_port.linear_gaussian_data(200, 4)
    est = build_nsf(theta, x)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        est.log_prob(theta[:3], x[:3])
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        NPE(device="cpu")
