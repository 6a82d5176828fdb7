"""Host logic of the tensor-core operand packing (pack.NsfLayout.tc_plan / RatioLayout.tc_plan):
the gather map must reproduce every linear of the network in the K-major no-swizzle wgmma layout
[K/4 slabs][N rows][4 floats], hi half then lo half (CPU only; the device side is
tests/test_nsf_tc_gpu.py / test_ratio_samplers_gpu.py)."""
import numpy as np
import pytest
import torch

from sbi_b200 import _lib as L
from sbi_b200.pack import NsfLayout, RatioLayout


def _unblock(block, N, K):
    """[K/4][N][4] -> dense (N, K)"""
    return block.reshape(K // 4, N, 4).transpose(1, 0, 2).reshape(N, K)


def _apply(src, params):
    out = np.zeros(src.shape, np.float64)
    hi = src >= 0
    lo = src <= -2
    out[hi] = params[src[hi]]
    out[lo] = -params[-2 - src[lo]]          # marks "lo" entries with the negated value
    return out


@pytest.mark.parametrize("D,C", [(10, 10), (2, 2), (5, 7), (16, 3)])
def test_nsf_tc_plan_reproduces_the_linears(D, C):
    lay = NsfLayout(D=D, C=C)
    plan = lay.tc_plan()
    assert plan is not None
    H, Hp, Cp, K0p, PR, NPAR = lay.H, lay.Hp, lay.Cp, lay.K0p, lay.PR, lay.NPAR
    rng = np.random.default_rng(0)
    params = rng.standard_normal(lay.n_params)
    vals = _apply(plan["src"], params)
    tab = plan["tab"].reshape(lay.T, L.SBI_NSF_TC_STRIDE)
    assert plan["stage_cap"] % 32 == 0 and plan["n_words"] == plan["src"].size
    KC0, nkc = H // 8, (H + C + 7) // 8 - H // 8
    for l in range(lay.T):
        lt = lay.layer_tab[l]
        n_id, n_tr = int(lt[L.L_NID]), int(lt[L.L_NTR])
        ns, kid8 = int(tab[l, 0]), int(tab[l, 1])
        assert kid8 == (n_id + 7) // 8 * 8 and ns == 1 + 3 * lay.NB + (n_tr + 1) // 2
        stages = [tab[l, 4 + 4 * s: 8 + 4 * s] for s in range(ns)]
        for off, nfl, N, aux in stages:
            assert nfl <= plan["stage_cap"] and nfl % 2 == 0
            hi, lo = vals[off: off + nfl // 2], vals[off + nfl // 2: off + nfl]
            assert np.array_equal(lo, -hi)                      # lo half mirrors the hi half's sources
        # initial layer: identity block then context block
        off, nfl, N, _ = stages[0]
        hi = vals[off: off + nfl // 2]
        w0 = params[int(lt[L.L_W0]):][: Hp * K0p].reshape(Hp, K0p)
        idb = _unblock(hi[: 64 * kid8], 64, kid8)
        assert np.array_equal(idb[:H, :n_id], w0[:H, Cp: Cp + n_id])
        assert not idb[H:].any() and not idb[:, n_id:].any()
        ctxb = _unblock(hi[64 * kid8:], 64, 8 * nkc)
        for c in range(C):
            assert np.array_equal(ctxb[:H, H - 8 * KC0 + c], w0[:H, c])
        assert np.count_nonzero(ctxb) <= H * C
        # blocks
        for b in range(lay.NB):
            t = L.L_BLK0 + 6 * b
            w1 = params[int(lt[t + 0]):][: Hp * Hp].reshape(Hp, Hp)
            w2 = params[int(lt[t + 2]):][: Hp * Hp].reshape(Hp, Hp)
            wc = params[int(lt[t + 4]):][: Hp * Cp].reshape(Hp, Cp)
            o_c, n_c, _, _ = stages[1 + 3 * b]
            o_1, n_1, _, _ = stages[2 + 3 * b]
            o_2, n_2, _, _ = stages[3 + 3 * b]
            gc = _unblock(vals[o_c: o_c + n_c // 2], 64, 8 * nkc)
            for c in range(C):
                assert np.array_equal(gc[:H, H - 8 * KC0 + c], wc[:H, c])
            d1 = _unblock(vals[o_1: o_1 + n_1 // 2], 64, 56)
            d2 = _unblock(vals[o_2: o_2 + n_2 // 2], 64, 56)
            assert np.array_equal(d1[:H, :H], w1[:H, :H]) and not d1[H:].any() and not d1[:, H:].any()
            assert np.array_equal(d2[:H, :H], w2[:H, :H]) and not d2[H:].any() and not d2[:, H:].any()
        # final-layer passes: 32 rows per spline feature
        wf = params[int(lt[L.L_WF]):][: n_tr * PR * Hp].reshape(n_tr * PR, Hp)
        seen = 0
        for off, nfl, N, aux in stages[1 + 3 * lay.NB:]:
            f0, nf = int(aux) & 0xffff, int(aux) >> 16
            assert f0 == seen and N == 32 * nf and 1 <= nf <= 2
            blk = _unblock(vals[off: off + nfl // 2], N, 56)
            for f in range(nf):
                assert np.array_equal(blk[32 * f: 32 * f + NPAR, :H], wf[(f0 + f) * PR: (f0 + f) * PR + NPAR, :H])
                assert not blk[32 * f + NPAR: 32 * (f + 1)].any()
            seen += nf
        assert seen == n_tr


@pytest.mark.parametrize("D,C", [(10, 10), (2, 2), (5, 7), (16, 3)])
def test_nsf_tc_bwd_plan_holds_the_transposed_linears(D, C):
    """Backward chain operands (pack.NsfLayout.tc_bwd_plan): B[n][k] = W[k][n] for every linear, in the
    order the backward sweep consumes them."""
    lay = NsfLayout(D=D, C=C)
    plan = lay.tc_bwd_plan()
    assert plan is not None
    H, Hp, Cp, K0p, PR, NPAR = lay.H, lay.Hp, lay.Cp, lay.K0p, lay.PR, lay.NPAR
    params = np.random.default_rng(2).standard_normal(lay.n_params)
    vals = _apply(plan["src"], params)
    tab = plan["tab"].reshape(lay.T, L.SBI_NSF_TC_STRIDE)
    for l in range(lay.T):
        lt = lay.layer_tab[l]
        n_id, n_tr = int(lt[L.L_NID]), int(lt[L.L_NTR])
        npass = (n_tr + 1) // 2
        assert int(tab[l, 0]) == npass + 2 * lay.NB + 1 and int(tab[l, 1]) == npass
        st = [tab[l, 4 + 4 * s: 8 + 4 * s] for s in range(int(tab[l, 0]))]
        for off, nfl, N, aux in st:
            assert nfl <= plan["stage_cap"]
            assert np.array_equal(vals[off + nfl // 2: off + nfl], -vals[off: off + nfl // 2])
        wf = params[int(lt[L.L_WF]):][: n_tr * PR * Hp].reshape(n_tr * PR, Hp)
        for p in range(npass):
            off, nfl, N, aux = st[p]
            nf = min(2, n_tr - 2 * p)
            assert N == 64 and aux == 4 * nf
            blk = _unblock(vals[off: off + nfl // 2], 64, 32 * nf)
            for f in range(nf):
                w = wf[(2 * p + f) * PR: (2 * p + f) * PR + NPAR, :H]            # (NPAR, H)
                assert np.array_equal(blk[:H, 32 * f: 32 * f + NPAR], w.T)
                assert not blk[:, 32 * f + NPAR: 32 * (f + 1)].any()
            assert not blk[H:].any()
        s = npass
        for b in range(lay.NB - 1, -1, -1):
            t = L.L_BLK0 + 6 * b
            for wo in (int(lt[t + 2]), int(lt[t + 0])):
                w = params[wo:][: Hp * Hp].reshape(Hp, Hp)
                off, nfl, N, aux = st[s]
                blk = _unblock(vals[off: off + nfl // 2], 64, 56)
                assert N == 64 and aux == 7 and np.array_equal(blk[:H, :H], w[:H, :H].T)
                assert not blk[H:].any() and not blk[:, H:].any()
                s += 1
        off, nfl, N, aux = st[s]
        w0 = params[int(lt[L.L_W0]):][: Hp * K0p].reshape(Hp, K0p)
        blk = _unblock(vals[off: off + nfl // 2], 16, 56)
        assert N == 16 and np.array_equal(blk[:n_id, :H], w0[:H, Cp: Cp + n_id].T)
        assert not blk[n_id:].any() and not blk[:, H:].any()


def test_nsf_tc_plan_rejects_what_the_kernel_does_not_instantiate():
    assert NsfLayout(D=4, C=3, H=32).tc_plan() is None          # hidden width
    assert NsfLayout(D=4, C=20).tc_plan() is None               # H + C > 64
    assert NsfLayout(D=20, C=4).tc_plan() is None               # D > 16 (register-resident LU)
    assert NsfLayout(D=4, C=3, KB=8).tc_plan() is None          # bin count


@pytest.mark.parametrize("Dt,Dx", [(10, 10), (1, 1), (4, 6)])
def test_ratio_tc_plan_reproduces_the_linears(Dt, Dx):
    lay = RatioLayout(Dt=Dt, Dx=Dx)
    plan = lay.tc_plan()
    assert plan is not None
    H, Hp, K0p, Dtp = lay.H, lay.Hp, lay.Dtp + lay.Dxp, lay.Dtp
    rng = np.random.default_rng(1)
    params = rng.standard_normal(lay.n_params)
    vals = _apply(plan["src"], params)
    tab = plan["tab"]
    ns, k0p8 = int(tab[0]), int(tab[1])
    assert ns == 2 + 2 * lay.NB and k0p8 == (Dt + Dx + 7) // 8 * 8
    st = [tab[4 + 4 * s: 8 + 4 * s] for s in range(ns)]
    w0 = params[int(lay.tab[L.R_W0]):][: Hp * K0p].reshape(Hp, K0p)
    b0 = _unblock(vals[st[0][0]: st[0][0] + st[0][1] // 2], 64, k0p8)
    assert np.array_equal(b0[:H, :Dt], w0[:H, :Dt]) and np.array_equal(b0[:H, Dt: Dt + Dx], w0[:H, Dtp: Dtp + Dx])
    assert not b0[H:].any() and not b0[:, Dt + Dx:].any()
    for b in range(lay.NB):
        for j in range(2):
            w = params[int(lay.tab[L.R_BLK0 + 4 * b + 2 * j]):][: Hp * Hp].reshape(Hp, Hp)
            o, n, N, _ = st[1 + 2 * b + j]
            blk = _unblock(vals[o: o + n // 2], 64, 56)
            assert N == 64 and np.array_equal(blk[:H, :H], w[:H, :H]) and not blk[H:].any()
    o, n, N, _ = st[-1]
    wf = params[int(lay.tab[L.R_WF]):][:Hp]
    blk = _unblock(vals[o: o + n // 2], 16, 56)
    assert N == 16 and np.array_equal(blk[0, :H], wf[:H]) and not blk[1:].any()
    assert RatioLayout(Dt=40, Dx=30).tc_plan() is None
