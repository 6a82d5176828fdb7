"""Launch-side tuning of the flow-matching weight pipeline (csrc/fm.cu `fm_tune`, exported as
`sbi_b200_fm_plan`): for every model shape the re-chunked plan keeps the kernels' invariants (chunk rows a
multiple of 4 and within the matrix, every chunk within a ring stage, 2..8 stages) and never turns a plan that
fits the 227 KB of shared memory into one that does not.  No device work."""
import ctypes as C
import itertools

import pytest

from sbi_b200 import _lib as L
from sbi_b200.pack import FmLayout

SMEM_MAX = 227 * 1024


def _plans(D, Cn, H, NL, TE):
    lib = L.load()
    lay = FmLayout(D=D, C=Cn, H=H, NL=NL, TE=TE)
    s = L.FmModel()
    lay.fill_struct(s, 2)
    out = []
    for kernel in range(3):
        v = (C.c_int32 * 10)()
        assert lib.sbi_b200_fm_plan(C.byref(s), kernel, v) == 0
        out.append(list(v))
    return lay, out


def _caller_smem(lay, kernel):
    """Shared memory of the caller's own plan (csrc/fm.cu fm_smem_layout restated)."""
    TM = 32 if kernel == 0 else 16
    train, trace = kernel == 1, kernel == 2
    Hp, Dp, Cp, TEp, NL = lay.Hp, lay.Dp, lay.Cp, lay.TEp, lay.NL
    rows = Dp + Cp + TEp + (0 if trace else Dp) + (2 * Hp if train or trace else 0) + 2 * Hp
    rows += (Hp if train or trace else 0) + ((NL + 1) if train else 1) * Hp + (NL if train or trace else 1) * Hp
    rows += Hp + Hp + (Hp if train else 0) + ((2 * NL + 3) // 4 * 4) + 32 + Dp + (2 * Hp if train else 0)
    rows += (NL * Hp + 2 * Hp + Hp + Hp + 1) if trace else 0
    fl = (rows * (TM + 4) + 31) // 32 * 32
    return (fl + 2 * lay.wcap) * 4 + 2 * 2 * 8 + 16


@pytest.mark.parametrize("H", [16, 50, 64, 100, 128])
def test_plans_keep_the_kernel_invariants(H):
    for D, Cn, NL, TE in itertools.product((1, 3, 20, 50), (1, 7, 20, 64), (2, 3, 5, 8), (16, 32)):
        lay, plans = _plans(D, Cn, H, NL, TE)
        for kernel, (nbuf, wcap, ri, rc, rm, rt, rh, ro, smem, rn) in enumerate(plans):
            for r, rowlen, nmax in ((ri, lay.Dp, lay.Hp), (rc, lay.Cp, lay.Hp), (rm, 2 * lay.Hp, lay.Hp),
                                    (rt, lay.TEp, lay.Hp), (rh, lay.Hp, lay.Hp), (ro, lay.Hp, lay.Dp)):
                assert r % 4 == 0 and 4 <= r <= nmax and r * rowlen <= wcap
            assert 2 <= nbuf <= 8 and wcap % 32 == 0 and rn in (1, 2)
            if _caller_smem(lay, kernel) <= SMEM_MAX - 1024:
                assert smem <= SMEM_MAX - 1024, (D, Cn, H, NL, TE, kernel, smem)


def test_default_network_plan():
    """posterior_flow_nn / posterior_score_nn defaults at dim 20 (BASELINE configs[3]): two stages, hidden layers
    in chunks of >= 48 rows for the training and divergence kernels, whole layers for the evaluation kernel."""
    lay, (ev, tr, dv) = _plans(20, 20, 100, 5, 32)
    assert ev[6] == 100 and tr[6] >= 48 and dv[6] >= 48
    for p in (ev, tr, dv):
        assert p[8] <= SMEM_MAX


def test_shared_memory_limit_per_kernel():
    """The largest hidden width each kernel fits at D = C = 20, num_layers = 5 (DESIGN.md §3.1): the 32-row
    forward takes H = 224, the 16-row loss / network VJP 124 and the forward + divergence 120, so evaluation fits
    models (H = 128) that training does not."""
    limits = [max(H for H in range(4, 400, 4) if _plans(20, 20, H, 5, 32)[1][k][8] <= SMEM_MAX) for k in range(3)]
    assert limits == [224, 124, 120]
