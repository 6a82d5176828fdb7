"""Packed parameter layout of the NSF kernels and its mapping to nflows' state_dict.

The kernels read ONE flat fp32 buffer.  Every matrix keeps PyTorch's native [out][in]
layout with the input dimension zero-padded to a multiple of 4 floats (16-byte rows for
cp.async.bulk and float4 shared-memory reads) and the output dimension padded to a multiple
of 4 with zero rows.  `NsfLayout` computes offsets, the per-layer descriptor table the
kernels index (include/sbi_b200.h, SBI_L_*), and, for every tensor of the reference
module (`net._transform._transforms.{i}...`, names as produced by the reference builder
sbi/neural_nets/net_builders/flow.py:333-460 on nflows 0.14), an index map
into the flat buffer, so a reference state_dict can be loaded / exported verbatim.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib as L


def round4(x: int) -> int:
    return (x + 3) & ~3


def round32(x: int) -> int:
    return (x + 31) & ~31


class _Alloc:
    """The running offset into the flat buffer and the index map of the reference tensors placed so far."""

    def __init__(self):
        self.off = 0
        self.index: Dict[str, np.ndarray] = {}

    def take(self, n: int) -> int:
        """Reserve n floats, rounded up to a multiple of 4; returns their offset."""
        o = self.off
        self.off += round4(n)
        return o

    def linear(self, name: str, tab: np.ndarray, slots, N: int, K: int, Kp: int, cols=None, rows=None):
        """Reserve the torch Linear `name` (N outputs, K inputs): its weight in rows of Kp floats, then its bias, with
        their offsets stored at tab[slots[0]] and tab[slots[1]].  Input k sits in column cols[k] (default k) and
        output n in row rows[n] (default n); both blocks hold the rows up to the last used one, rounded up to 4."""
        cols = np.arange(K) if cols is None else cols
        rows = np.arange(N) if rows is None else rows
        n_rows = round4(int(rows[-1]) + 1)
        o = tab[slots[0]] = self.take(n_rows * Kp)
        self.index[name + ".weight"] = o + rows[:, None] * Kp + cols[None, :]
        o = tab[slots[1]] = self.take(n_rows)
        self.index[name + ".bias"] = o + rows


def _plan_ring(cap: int, mats, extra=()):
    """Weight-ring chunking.  For each matrix (row length, row count): the rows per chunk, as many whole rows as fit
    in `cap` floats, a multiple of 4, at least 4 and at most the row count.  Returns those and the ring slot size
    wcap: the largest chunk or `extra` term in floats, rounded up to 32."""
    rpc = [max(4, min(nmax, (cap // rowlen) & ~3)) for rowlen, nmax in mats]
    used = max([r * rowlen for r, (rowlen, _) in zip(rpc, mats)] + list(extra))
    return rpc, round32(used)


def _made_masks(D: int, H: int, out_mult: int):
    """nflows MADE with sequential degrees (transforms/made.py) on D inputs, H hidden units and out_mult outputs per
    input: the input, hidden and output degrees and the (H, D) initial, (H, H) hidden and (out_mult*D, H) final
    masks."""
    in_deg = np.arange(1, D + 1)
    max_, min_ = max(1, D - 1), min(1, D - 1)
    hid_deg = np.arange(H) % max_ + min_
    out_deg = np.repeat(in_deg, out_mult)
    m_init = (hid_deg[:, None] >= in_deg[None, :]).astype(np.float32)
    m_hid = (hid_deg[:, None] >= hid_deg[None, :]).astype(np.float32)
    m_out = (out_deg[:, None] > hid_deg[None, :]).astype(np.float32)
    return in_deg, hid_deg, out_deg, m_init, m_hid, m_out


def _add_mask(lay, name: str, mask: np.ndarray, degrees: np.ndarray):
    """MADE's masked linear `name`: the packed weight holds W * mask; the module's `mask` / `degrees` buffers."""
    lay._weight_masks[name + ".weight"] = mask
    lay.buffers[name + ".mask"] = torch.as_tensor(mask)
    lay.buffers[name + ".degrees"] = torch.as_tensor(degrees)


def _residual_blocks(a: _Alloc, lay, prefix: str, tab: np.ndarray, hidden_mask=None):
    """The `{prefix}blocks.{b}` of an nflows ResidualNet with a context layer: linear_layers.0, linear_layers.1 and
    context_layer at table fields L_BLK0 + 6b .. L_BLK0 + 6b + 5.  hidden_mask: (mask, degrees) of MADE's masked
    linear_layers."""
    for b in range(lay.NB):
        pb = prefix + f"blocks.{b}."
        t = L.L_BLK0 + 6 * b
        for j in range(2):
            a.linear(pb + f"linear_layers.{j}", tab, (t + 2 * j, t + 2 * j + 1), lay.H, lay.H, lay.Hp)
            if hidden_mask is not None:
                _add_mask(lay, pb + f"linear_layers.{j}", *hidden_mask)
        a.linear(pb + "context_layer", tab, (t + 4, t + 5), lay.H, lay.C, lay.Cp)


def _tc_block(N: int, K: int, fill):
    """One K-major no-swizzle wgmma operand block [K/4 slabs][N rows][4 floats], flattened.
    fill(n, k) -> the parameter index of element (n, k), or -1 for a zero."""
    blk = np.full((K // 4, N, 4), -1, np.int64)
    n = np.arange(N)[:, None] + 0 * np.arange(K)[None, :]
    k = np.arange(K)[None, :] + 0 * np.arange(N)[:, None]
    blk[k // 4, n, k % 4] = fill(n, k)
    return blk.reshape(-1)


def _tc_assemble(rows):
    """Gather map and stage table of a wgmma operand plan (include/sbi_b200.h `sbi_nsf_tc`).  rows: per table row
    (layer) its second header word and its stages (hi, N, aux), hi the gather map of the stage's hi half; word 0 is
    the stage count.  A stage is its hi half, then its lo half (-2 - index where hi holds a parameter).
    Returns dict(src=int32 (n_words,), tab=int32 (rows * STRIDE,), stage_cap=int, n_words=int)."""
    tab = np.zeros((len(rows), L.SBI_NSF_TC_STRIDE), np.int32)
    chunks, off, stage_cap = [], 0, 0
    for r, (word1, stages) in enumerate(rows):
        tab[r, 0], tab[r, 1] = len(stages), word1
        for s, (hi, N, aux) in enumerate(stages):
            nfl = 2 * hi.size
            tab[r, 4 + 4 * s: 8 + 4 * s] = (off, nfl, N, aux)
            chunks += [hi, np.where(hi >= 0, -2 - hi, -1)]
            off += nfl
            stage_cap = max(stage_cap, nfl)
    return dict(src=np.concatenate(chunks).astype(np.int32), tab=tab.reshape(-1),
                stage_cap=round32(stage_cap), n_words=off)


class _LayoutOps:
    """Base of the packed layouts: pack / unpack between reference-named tensors and the flat kernel buffer.
    `_weight_masks` holds, for masked (MADE) weights, the 0/1 mask: the flat buffer stores W*M, the masked-out raw
    values are kept aside (`raw`) only so that state_dict() round-trips exactly.  Subclasses set `n_params`, `index`
    and `buffers`."""

    family: str                  # the estimator family the layout belongs to
    _tables = ("tab",)           # the attributes `tables()` returns
    _weight_masks: Dict[str, np.ndarray] = {}      # shared empty default: masked layouts assign their own

    def _wm(self) -> Dict[str, np.ndarray]:
        """The weight masks, {reference weight name: 0/1 mask}; empty unless the layout has masked weights."""
        return self._weight_masks

    def trainable_mask(self) -> torch.Tensor:
        m = torch.zeros(self.n_params, dtype=torch.uint8)
        for k, v in self.index.items():
            ix = torch.as_tensor(v.reshape(-1))
            if k in self._weight_masks:
                m[ix] = torch.as_tensor(self._weight_masks[k].reshape(-1)).to(torch.uint8)
            else:
                m[ix] = 1
        return m

    def pack(self, state: Dict[str, torch.Tensor], out: torch.Tensor = None,
             raw_out: torch.Tensor = None) -> torch.Tensor:
        """Reference-named tensors -> flat buffer (on out's device if given)."""
        flat = torch.zeros(self.n_params, dtype=torch.float32) if out is None else out
        for k, ix in self.index.items():
            src = state[k].detach().to(dtype=torch.float32, device=flat.device).reshape(-1)
            pos = torch.as_tensor(ix.reshape(-1), device=flat.device)
            if k in self._weight_masks:
                mk = torch.as_tensor(self._weight_masks[k].reshape(-1), dtype=torch.float32, device=flat.device)
                if raw_out is not None:
                    raw_out[pos] = src * (1 - mk)
                src = src * mk
            flat[pos] = src
        return flat

    def unpack(self, flat: torch.Tensor, raw: torch.Tensor = None) -> Dict[str, torch.Tensor]:
        out = {}
        for k, ix in self.index.items():
            pos = torch.as_tensor(ix.reshape(-1), device=flat.device)
            t = flat.detach()[pos]
            if raw is not None and k in self._weight_masks:
                t = t + raw[pos]
            out[k] = t.reshape(ix.shape).clone()
        return out

    def num_real_params(self) -> int:
        return int(sum(v.size for v in self.index.values()))

    def tables(self):
        """The int32 index tables the model struct points to, in the order of its table fields."""
        return tuple(getattr(self, name).reshape(-1).astype(np.int32) for name in self._tables)

    def tc_plan(self):
        """The operand plan of the family's wgmma evaluation kernel, or None if there is none for this model."""
        return None

    def tc_bwd_plan(self):
        """The operand plan of the transposed linears for the wgmma training kernel, or None."""
        return None

    def load_buffers(self, incoming: Dict[str, torch.Tensor]):
        """Adopt structural buffers of a loaded state_dict that are data rather than architecture.  Returns None when
        the index tables did not change."""
        return None


class _NsfKernelLayout(_LayoutOps):
    """The layouts that run on the NSF kernels (include/sbi_b200.h `sbi_nsf_model`): the weight ring and the
    common struct fields.  Subclasses set the head fields of the struct."""

    _tables = ("layer_tab", "feat_tab")

    def _plan_nsf_ring(self):
        """Ring chunks of the initial ([., K0p]), hidden ([., Hp]) and context-gated ([., Hp + Cp]) matrices, and of
        the final layer: nf_chunk features of PR x Hp floats each."""
        Hp, Cp, K0p, PR = self.Hp, self.Cp, self.K0p, self.PR
        cap = max(self.wcap_target, 4 * K0p, 4 * (Hp + Cp), PR * Hp)
        self.nf_chunk = max(1, min(self.TRmax, cap // (PR * Hp)))
        (self.rpc0, self.rpc1, self.rpc2), self.wcap = _plan_ring(
            cap, [(K0p, Hp), (Hp, Hp), (Hp + Cp, Hp)], [self.nf_chunk * PR * Hp])

    def fill_struct(self, s: "L.NsfModel", nbuf: int):
        s.D, s.C, s.H, s.NB, s.KB, s.T = self.D, self.C, self.H, self.NB, self.KB, self.T
        s.Dp, s.Cp, s.IDp, s.Hp, s.PR = self.Dp, self.Cp, self.IDp, self.Hp, self.PR
        s.TRmax, s.nf_chunk = self.TRmax, self.nf_chunk
        s.rpc0, s.rpc1, s.rpc2 = self.rpc0, self.rpc1, self.rpc2
        s.wcap, s.nbuf, s.n_params = self.wcap, nbuf, self.n_params
        s.min_bw = s.min_bh = s.min_d = 1e-3
        return s


@dataclass
class NsfLayout(_NsfKernelLayout):
    D: int
    C: int
    H: int = 50
    NB: int = 2
    KB: int = 10
    T: int = 5
    tail_bound: float = 3.0
    zscore_input: bool = True
    zscore_cond: bool = True
    embed_is_identity: bool = True
    wcap_target: int = int(__import__('os').environ.get('SBI_B200_WCAP', 4096))

    family = "nsf"

    def __post_init__(self):
        D, C, H, NB, KB, T = self.D, self.C, self.H, self.NB, self.KB, self.T
        if D < 2:
            raise NotImplementedError("NSF kernels need input dim >= 2")
        if NB > L.SBI_NSF_MAX_BLOCKS:
            raise ValueError(f"num_blocks <= {L.SBI_NSF_MAX_BLOCKS}")
        self.Dp, self.Cp, self.Hp = round4(D), round4(C), round4(H)
        self.NPAR = 3 * KB - 1
        self.PR = round4(self.NPAR)
        # alternating masks, reference: torchutils.py:396-410 / flow.py:396-397
        self.id_feats: List[np.ndarray] = []
        self.tr_feats: List[np.ndarray] = []
        for i in range(T):
            mask = np.zeros(D, np.int64)
            mask[(0 if i % 2 == 0 else 1)::2] = 1
            self.tr_feats.append(np.nonzero(mask > 0)[0])
            self.id_feats.append(np.nonzero(mask <= 0)[0])
        self.IDp = round4(max(len(f) for f in self.id_feats))
        self.TRmax = max(len(f) for f in self.tr_feats)
        self.K0p = self.Cp + self.IDp
        self._plan_nsf_ring()

        a = _Alloc()
        tab = np.zeros((T, L.SBI_NSF_LAYER_STRIDE), np.int32)
        feat = []
        ntri = D * (D - 1) // 2
        base = 1 if self.zscore_input else 0
        self.buffers: Dict[str, torch.Tensor] = {}
        for l in range(T):
            idf, trf = self.id_feats[l], self.tr_feats[l]
            n_id, n_tr = len(idf), len(trf)
            pc = f"net._transform._transforms.{base + 2 * l}."
            pl = f"net._transform._transforms.{base + 2 * l + 1}."
            t = tab[l]
            t[L.L_NID], t[L.L_NTR], t[L.L_FEAT] = n_id, n_tr, len(feat)
            feat += list(idf) + list(trf)
            self.buffers[pc + "identity_features"] = torch.as_tensor(idf)
            self.buffers[pc + "transform_features"] = torch.as_tensor(trf)
            # initial layer: nflows columns [id | ctx] -> packed columns [ctx | pad | id | pad]
            a.linear(pc + "transform_net.initial_layer", t, (L.L_W0, L.L_B0), H, n_id + C, self.K0p,
                     cols=np.concatenate([self.Cp + np.arange(n_id), np.arange(C)]))
            _residual_blocks(a, self, pc + "transform_net.", t)
            # final layer: feature f owns packed rows f*PR .. f*PR+NPAR-1
            prow = (np.arange(n_tr)[:, None] * self.PR + np.arange(self.NPAR)[None, :]).reshape(-1)
            a.linear(pc + "transform_net.final_layer", t, (L.L_WF, L.L_BF), n_tr * self.NPAR, H, self.Hp, rows=prow)
            # LULinear
            t[L.L_HAS_LU] = 1
            for slot, name, n in ((L.L_LU_LOWER, "lower_entries", ntri), (L.L_LU_UPPER, "upper_entries", ntri),
                                  (L.L_LU_DIAG, "unconstrained_upper_diag", D), (L.L_LU_BIAS, "bias", D)):
                o = t[slot] = a.take(n)
                a.index[pl + name] = o + np.arange(n)
        self.n_params = a.off
        self.index = a.index
        self.layer_tab = tab
        self.feat_tab = np.asarray(feat, np.int32)
        self.edge_raw = float(np.log(np.exp(1 - 1e-3) - 1))

    def fill_struct(self, s: "L.NsfModel", nbuf: int):
        super().fill_struct(s, nbuf)
        s.tail_bound, s.inv_sqrt_h, s.edge_raw = self.tail_bound, 1.0 / math.sqrt(self.H), self.edge_raw
        s.head, s.M, s.mog_eps, s.cond_mlp = 0, 0, 0.0, 0
        return s

    # ------------------------------------------------------------- tensor-core operand plan
    def tc_plan(self):
        """Gather map + stage table for the wgmma evaluation path (include/sbi_b200.h,
        `sbi_nsf_tc`; kernel sbi_b200/csrc/nsf_tc.cu), or None when the model is outside what
        that kernel instantiates.

        Every linear of the conditioner (nflows ResidualNet) becomes one or two K-major
        no-swizzle (interleaved) wgmma operand blocks [K/4 slabs][N rows][4 floats].  The hidden operand's
        columns are [hidden (H) | context (C) | 0] so that the context never needs its own
        staging: the GLU gate reads the K-steps that cover columns H..H+C-1.
        Returns dict(src=int32 (n_words,), tab=int32 (T*STRIDE,), stage_cap=int, n_words=int).
        """
        D, C, H, NB, T = self.D, self.C, self.H, self.NB, self.T
        if H != 50 or self.KB != 10 or H + C > 64 or self.IDp > 48 or self.PR > 32 or D > 16:
            return None
        Hp, Cp, K0p, PR, NPAR = self.Hp, self.Cp, self.K0p, self.PR, self.NPAR
        HP8 = (H + 7) & ~7
        KC0 = H // 8
        nkc = (H + C + 7) // 8 - KC0

        def ctx_block(woff, rowlen):
            def fill(n, k):
                c = 8 * KC0 + k - H
                ok = (n < H) & (c >= 0) & (c < C)
                return np.where(ok, woff + n * rowlen + np.clip(c, 0, max(C - 1, 0)), -1)
            return _tc_block(64, 8 * nkc, fill)

        def hidden_block(woff, N, rowmap):
            """rowmap(n) -> (valid, packed row index) of the [.,Hp] weight matrix"""
            def fill(n, k):
                valid, row = rowmap(n)
                ok = valid & (k < H)
                return np.where(ok, woff + row * Hp + np.minimum(k, H - 1), -1)
            return _tc_block(N, HP8, fill)

        rows = []
        for l in range(T):
            lt = self.layer_tab[l]
            n_id, n_tr = int(lt[L.L_NID]), int(lt[L.L_NTR])
            kid8 = (n_id + 7) & ~7
            w0 = int(lt[L.L_W0])

            def fill_id(n, k, w0=w0, n_id=n_id):
                ok = (n < H) & (k < n_id)
                return np.where(ok, w0 + n * K0p + Cp + np.minimum(k, max(n_id - 1, 0)), -1)

            stages = [(np.concatenate([_tc_block(64, kid8, fill_id), ctx_block(w0, K0p)]), 64, 0)]
            ident = lambda n: (n < H, np.minimum(n, H - 1))
            for b in range(NB):
                t = L.L_BLK0 + 6 * b
                w1, w2, wc = int(lt[t + 0]), int(lt[t + 2]), int(lt[t + 4])
                stages.append((ctx_block(wc, Cp), 64, 0))
                stages.append((hidden_block(w1, 64, ident), 64, 0))
                stages.append((hidden_block(w2, 64, ident), 64, 0))
            wf = int(lt[L.L_WF])
            f0 = 0
            while f0 < n_tr:
                nf = min(2, n_tr - f0)

                def rowmap(n, f0=f0, nf=nf):
                    f, i = n // 32, n % 32
                    valid = (f < nf) & (i < NPAR)
                    return valid, np.where(valid, (f0 + f) * PR + i, 0)

                stages.append((hidden_block(wf, 32 * nf, rowmap), 32 * nf, f0 | (nf << 16)))
                f0 += nf
            if len(stages) > L.SBI_NSF_TC_MAX_STAGES:
                return None
            rows.append((kid8, stages))
        return _tc_assemble(rows)

    def tc_bwd_plan(self):
        """Gather map + stage table of the TRANSPOSED linears for the wgmma training kernel's
        input-gradient chain (kernel sbi_b200/csrc/nsf_vjp_tc.cu): dX = dY W needs, as the B operand
        [N = in-features][K = out-features] in the same K-major no-swizzle layout, B[n][k] = W[k][n].
        Stages of a layer in the order the backward sweep uses them (aux = number of K-steps):
            final layer, one pass per <= 2 spline features:  N = 64 (hidden), K = 32 * nf
            per block b = NB-1 .. 0:  W2^T (N = 64, K = 56),  W1^T (N = 64, K = 56)
            initial layer, identity-feature columns only:  N = 16, K = 56
        Same return format as tc_plan (the context columns are not needed: training never asks for
        the condition's gradient on this path)."""
        H, NB, T = self.H, self.NB, self.T
        if self.tc_plan() is None or self.IDp > 16:
            return None
        Hp, Cp, K0p, PR, NPAR = self.Hp, self.Cp, self.K0p, self.PR, self.NPAR
        HP8 = (H + 7) & ~7
        rows = []
        for l in range(T):
            lt = self.layer_tab[l]
            n_id, n_tr = int(lt[L.L_NID]), int(lt[L.L_NTR])
            stages = []
            wf = int(lt[L.L_WF])
            f0 = 0
            while f0 < n_tr:
                nf = min(2, n_tr - f0)

                def fill_f(n, k, f0=f0, nf=nf):
                    f, i = k // 32, k % 32
                    ok = (n < H) & (f < nf) & (i < NPAR)
                    return np.where(ok, wf + ((f0 + np.minimum(f, nf - 1)) * PR + np.minimum(i, NPAR - 1)) * Hp
                                    + np.minimum(n, H - 1), -1)

                stages.append((_tc_block(64, 32 * nf, fill_f), 64, 4 * nf))
                f0 += nf
            for b in range(NB - 1, -1, -1):
                t = L.L_BLK0 + 6 * b
                for w in (int(lt[t + 2]), int(lt[t + 0])):          # W2 then W1

                    def fill_h(n, k, w=w):
                        ok = (n < H) & (k < H)
                        return np.where(ok, w + np.minimum(k, H - 1) * Hp + np.minimum(n, H - 1), -1)

                    stages.append((_tc_block(64, HP8, fill_h), 64, HP8 // 8))
            w0 = int(lt[L.L_W0])

            def fill_0(n, k, w0=w0, n_id=n_id):
                ok = (n < n_id) & (k < H)
                return np.where(ok, w0 + np.minimum(k, H - 1) * K0p + Cp + np.minimum(n, max(n_id - 1, 0)), -1)

            stages.append((_tc_block(16, HP8, fill_0), 16, HP8 // 8))
            rows.append(((n_tr + 1) // 2, stages))
        return _tc_assemble(rows)


@dataclass
class Nsf1dLayout(_NsfKernelLayout):
    """Packed layout of the ONE-dimensional neural spline flow (flow.py:401-432 with x_numel == 1): T spline
    transforms of the single feature whose 3K-1 parameters come from a context-only MLP (`ContextSplineMap`,
    flow.py:1419-1478: Linear -> ReLU -> hidden_layers x [one shared Linear -> ReLU] -> Linear), no LULinear.
    Runs on the NSF kernels (`sbi_nsf_model` with cond_mlp = 1, NB = hidden_layers, no identity features)."""
    C: int
    H: int = 50
    NB: int = 1                  # hidden_layers_spline_context
    KB: int = 10
    T: int = 5
    tail_bound: float = 3.0
    zscore_input: bool = True
    zscore_cond: bool = True
    embed_is_identity: bool = True
    wcap_target: int = 4096
    D: int = 1

    family = "nsf"

    def __post_init__(self):
        C, H, NB, KB, T = self.C, self.H, self.NB, self.KB, self.T
        if NB < 0 or NB > L.SBI_NSF_MAX_BLOCKS:
            raise ValueError(f"0 <= hidden_layers_spline_context <= {L.SBI_NSF_MAX_BLOCKS}")
        self.Dp, self.Cp, self.Hp = 4, round4(C), round4(H)
        self.NPAR = 3 * KB - 1
        self.PR = round4(self.NPAR)
        if self.PR > self.Hp:
            raise ValueError("hidden_features must be >= the padded spline parameter count")
        self.IDp, self.TRmax, self.K0p = 0, 1, self.Cp
        self._plan_nsf_ring()
        Hp = self.Hp
        a = _Alloc()
        tab = np.zeros((T, L.SBI_NSF_LAYER_STRIDE), np.int32)
        self.buffers: Dict[str, torch.Tensor] = {}
        base = 1 if self.zscore_input else 0
        for l in range(T):
            pc = f"net._transform._transforms.{base + l}."
            pn = pc + "transform_net.spline_predictor."
            t = tab[l]
            t[L.L_NID], t[L.L_NTR], t[L.L_FEAT] = 0, 1, l
            self.buffers[pc + "identity_features"] = torch.zeros(0, dtype=torch.int64)
            self.buffers[pc + "transform_features"] = torch.zeros(1, dtype=torch.int64)
            a.linear(pn + "0", t, (L.L_W0, L.L_B0), H, C, self.Cp)
            ow = t[L.L_BLK0] = a.take(Hp * Hp)
            ob = t[L.L_BLK0 + 1] = a.take(Hp)
            for k in range(NB):      # nn.Sequential lists the shared module once per position
                a.index[pn + f"{2 + 2 * k}.weight"] = ow + np.arange(H)[:, None] * Hp + np.arange(H)[None, :]
                a.index[pn + f"{2 + 2 * k}.bias"] = ob + np.arange(H)
            a.linear(pn + f"{2 + 2 * NB}", t, (L.L_WF, L.L_BF), self.NPAR, H, Hp)
            t[L.L_HAS_LU] = 0
        self.n_params = a.off
        self.index = a.index
        self.layer_tab = tab
        self.feat_tab = np.zeros(T, np.int32)            # layer l: no identity features, transformed feature 0
        self.edge_raw = float(np.log(np.exp(1 - 1e-3) - 1))

    def num_real_params(self) -> int:
        return int(len({int(i) for v in self.index.values() for i in v.reshape(-1)}))

    def fill_struct(self, s: "L.NsfModel", nbuf: int):
        super().fill_struct(s, nbuf)
        s.tail_bound, s.inv_sqrt_h, s.edge_raw = self.tail_bound, 1.0 / math.sqrt(self.H), self.edge_raw
        s.head, s.M, s.mog_eps, s.cond_mlp = 0, 0, 0.0, 1
        return s


@dataclass
class MadeLayout(_NsfKernelLayout):
    """Packed layout of sbi's `made` density estimator (flow.py:37-112): ONE masked residual network
    (nflows MixtureOfGaussiansMADE behind sbi's MADEMoGWrapper, nn_utils.py:133-201: `features + 1`
    inputs with a dummy first feature) emitting, per feature, num_mixture_components x (logit, mean,
    unconstrained std).  The network is structurally the NSF conditioner (initial linear on
    [context | inputs], residual blocks with GLU context gates, final linear), so it runs on the NSF
    kernels (include/sbi_b200.h `sbi_nsf_model` with head = SBI_NSF_MOG): masks are folded into the
    packed weights, every feature is both a conditioner input and an output, T = 1, no LU.
    `D` here is the NETWORK's feature count (the estimator's input dim + 1)."""
    D: int
    C: int
    H: int = 50
    NB: int = 5
    M: int = 10
    epsilon: float = 1e-2
    zscore_input: bool = True
    zscore_cond: bool = True
    embed_is_identity: bool = True
    wcap_target: int = 4096

    family = "made"

    def __post_init__(self):
        D, C, H, NB, M = self.D, self.C, self.H, self.NB, self.M
        if NB > L.SBI_NSF_MAX_BLOCKS:
            raise ValueError(f"num_blocks <= {L.SBI_NSF_MAX_BLOCKS}")
        if not (1 <= M <= 16):
            raise ValueError("the mixture code keeps <= 16 components in registers")
        self.T, self.KB = 1, 0
        self.Dp, self.Cp, self.Hp = round4(D), round4(C), round4(H)
        self.NPAR = 3 * M
        self.PR = round4(self.NPAR)
        self.IDp = round4(D)
        self.TRmax = D
        self.K0p = self.Cp + self.IDp
        self._plan_nsf_ring()
        Hp, Cp, K0p = self.Hp, self.Cp, self.K0p
        _, hid_deg, out_deg, m_init, m_hid, m_out = _made_masks(D, H, 3 * M)

        a = _Alloc()
        tab = np.zeros((1, L.SBI_NSF_LAYER_STRIDE), np.int32)
        t = tab[0]
        self._weight_masks: Dict[str, np.ndarray] = {}
        self.buffers: Dict[str, torch.Tensor] = {}
        pm = "net._distribution._made."
        t[L.L_NID], t[L.L_NTR], t[L.L_FEAT] = D, D, 0
        # initial layer: packed columns [ctx | pad | inputs | pad]; MADE's context_layer supplies the ctx columns
        o = t[L.L_W0] = a.take(Hp * K0p)
        a.index[pm + "initial_layer.weight"] = o + np.arange(H)[:, None] * K0p + (Cp + np.arange(D))[None, :]
        _add_mask(self, pm + "initial_layer", m_init, hid_deg)
        a.index[pm + "context_layer.weight"] = o + np.arange(H)[:, None] * K0p + np.arange(C)[None, :]
        o = t[L.L_B0] = a.take(Hp)
        a.index[pm + "initial_layer.bias"] = o + np.arange(H)
        o = t[L.L_BC0] = a.take(Hp)
        a.index[pm + "context_layer.bias"] = o + np.arange(H)
        _residual_blocks(a, self, pm, t, hidden_mask=(m_hid, hid_deg))
        # final layer: feature f owns packed rows f*PR .. f*PR + 3M - 1 (nflows row f*3M + 3m + k)
        prow = (np.arange(D)[:, None] * self.PR + np.arange(self.NPAR)[None, :]).reshape(-1)
        a.linear(pm + "final_layer", t, (L.L_WF, L.L_BF), D * self.NPAR, H, Hp, rows=prow)
        _add_mask(self, pm + "final_layer", m_out, out_deg)
        t[L.L_HAS_LU] = 0
        self.n_params = a.off
        self.index = a.index
        self.layer_tab = tab
        self.feat_tab = np.asarray(list(range(D)) * 2, np.int32)

    def fill_struct(self, s: "L.NsfModel", nbuf: int):
        super().fill_struct(s, nbuf)
        s.KB = 2
        s.tail_bound, s.inv_sqrt_h, s.edge_raw = 1.0, 1.0, 0.0
        s.head, s.M, s.mog_eps, s.cond_mlp = 1, self.M, self.epsilon, 0
        return s


@dataclass
class MafLayout(_LayoutOps):
    """Packed layout of the MAF kernels (include/sbi_b200.h `sbi_maf_model`), mapping the tensors of
    the reference module built by sbi/neural_nets/net_builders/flow.py:115-209 on
    nflows 0.14 (MaskedAffineAutoregressiveTransform(MADE) + RandomPermutation per layer)."""
    D: int
    C: int
    H: int = 50
    NB: int = 2
    T: int = 5
    perms: List[np.ndarray] = None       # permutation of each layer (RandomPermutation buffer)
    zscore_input: bool = True
    zscore_cond: bool = True
    embed_is_identity: bool = True
    scale_softplus: bool = True          # softplus(s)+1e-3 (see oracle/nflows_port/transforms/autoregressive.py)
    wcap_target: int = 4096
    # element-wise transform: "affine" (maf) or "rqs" (maf_rqs, flow.py:212-330; linear tails)
    head: str = "affine"
    KB: int = 10
    tail_bound: float = 3.0
    min_bin_width: float = 1e-3
    min_bin_height: float = 1e-3
    min_derivative: float = 1e-3

    family = "maf"
    _tables = ("layer_tab", "perm_tab")

    def __post_init__(self):
        D, C, H, NB, T = self.D, self.C, self.H, self.NB, self.T
        if NB > 8:
            raise ValueError("num_blocks <= 8")
        if self.head not in ("affine", "rqs"):
            raise ValueError(self.head)
        if self.head == "rqs" and not (2 <= self.KB <= 16):
            raise ValueError("the spline code keeps <= 16 bins in registers")
        self.OUTM = 2 if self.head == "affine" else 3 * self.KB - 1
        self.Dp, self.Cp, self.Hp = round4(D), round4(C), round4(H)
        self.OUTp = round4(self.OUTM * D)
        Hp, Dp, Cp = self.Hp, self.Dp, self.Cp
        cap = max(self.wcap_target, 4 * (Dp + Cp), 4 * Hp)
        (self.rpc0, self.rpc1, self.rpcf), self.wcap = _plan_ring(
            cap, [(Dp + Cp, Hp), (Hp, Hp), (Hp, self.OUTp)], [4 * Cp, 4 * Dp])
        in_deg, hid_deg, out_deg, m_init, m_hid, m_out = _made_masks(D, H, self.OUTM)
        self.degrees = dict(input=in_deg, hidden=hid_deg, output=out_deg)

        if self.perms is None:
            self.perms = [np.arange(D) for _ in range(T)]
        a = _Alloc()
        tab = np.zeros((T, L.SBI_MAF_LAYER_STRIDE), np.int32)
        self._weight_masks: Dict[str, np.ndarray] = {}
        self.buffers: Dict[str, torch.Tensor] = {}
        base = 1 if self.zscore_input else 0
        for l in range(T):
            pa = f"net._transform._transforms.{base + 2 * l}.autoregressive_net."
            pp = f"net._transform._transforms.{base + 2 * l + 1}."
            t = tab[l]
            t[L.M_PERM] = 2 * D * l                      # the perm table holds (perm, inverse) per layer
            self.buffers[pp + "_permutation"] = torch.as_tensor(np.asarray(self.perms[l], np.int64))
            a.linear(pa + "initial_layer", t, (L.M_W0, L.M_B0), H, D, Dp)
            _add_mask(self, pa + "initial_layer", m_init, hid_deg)
            a.linear(pa + "context_layer", t, (L.M_WC, L.M_BC), H, C, Cp)
            for b in range(NB):
                a.linear(pa + f"blocks.{b}.linear", t, (L.M_BLK0 + 2 * b, L.M_BLK0 + 2 * b + 1), H, H, Hp)
                _add_mask(self, pa + f"blocks.{b}.linear", m_hid, hid_deg)
            a.linear(pa + "final_layer", t, (L.M_WF, L.M_BF), self.OUTM * D, H, Hp)
            _add_mask(self, pa + "final_layer", m_out, out_deg)
        self.n_params = a.off
        self.index = a.index
        self.layer_tab = tab
        self.perm_tab = self._perm_table()

    def _perm_table(self):
        return np.asarray([i for p in self.perms for i in (*p, *np.argsort(p))], np.int32)

    def load_buffers(self, incoming: Dict[str, torch.Tensor]):
        """Adopt the permutations of a loaded reference state_dict (RandomPermutation buffers are
        drawn at construction, so they are data, not architecture).  Returns the new perm table."""
        base = 1 if self.zscore_input else 0
        changed = False
        for l in range(self.T):
            key = f"net._transform._transforms.{base + 2 * l + 1}._permutation"
            if key in incoming:
                perm = incoming[key].detach().cpu().numpy().astype(np.int64)
                if perm.shape != (self.D,) or sorted(perm.tolist()) != list(range(self.D)):
                    raise ValueError(f"{key}: not a permutation of {self.D} features")
                if not np.array_equal(perm, self.perms[l]):
                    changed = True
                self.perms[l] = perm
                self.buffers[key] = torch.as_tensor(perm)
        self.perm_tab = self._perm_table()
        return self.perm_tab if changed else None

    def fill_struct(self, s: "L.MafModel", nbuf: int):
        s.D, s.C, s.H, s.NB, s.T = self.D, self.C, self.H, self.NB, self.T
        s.Dp, s.Cp, s.Hp, s.OUTp = self.Dp, self.Cp, self.Hp, self.OUTp
        s.rpc0, s.rpc1, s.rpcf = self.rpc0, self.rpc1, self.rpcf
        s.wcap, s.nbuf, s.n_params = self.wcap, nbuf, self.n_params
        s.scale_softplus = 1 if self.scale_softplus else 0
        s.head, s.KB, s.OUTM = (0 if self.head == "affine" else 1), self.KB, self.OUTM
        s.tail_bound, s.min_w, s.min_h, s.min_d = (self.tail_bound, self.min_bin_width, self.min_bin_height,
                                                   self.min_derivative)
        s.isq = 1.0     # nflows' MADE has no `hidden_features` attribute: no 1/sqrt(H) logit scaling here
        return s


@dataclass
class RatioLayout(_LayoutOps):
    """Packed layout of the NRE `resnet` classifier (include/sbi_b200.h `sbi_ratio_model`): nflows
    ResidualNet(in=Dt+Dx, out=1, hidden, context=None, num_blocks) as built by
    sbi/neural_nets/net_builders/classifier.py:172-235."""
    Dt: int
    Dx: int
    H: int = 50
    NB: int = 2
    wcap_target: int = 4096

    family = "ratio"

    def __post_init__(self):
        Dt, Dx, H, NB = self.Dt, self.Dx, self.H, self.NB
        self.Dtp, self.Dxp, self.Hp = round4(Dt), round4(Dx), round4(H)
        K0p, Hp = self.Dtp + self.Dxp, self.Hp
        cap = max(self.wcap_target, 4 * K0p, 4 * Hp)
        (self.rpc0, self.rpc1), self.wcap = _plan_ring(cap, [(K0p, Hp), (Hp, Hp)], [4 * Hp])
        a = _Alloc()
        tab = np.zeros(4 + 4 * 8, np.int32)
        a.linear("net.initial_layer", tab, (L.R_W0, L.R_B0), H, Dt + Dx, K0p,
                 cols=np.concatenate([np.arange(Dt), self.Dtp + np.arange(Dx)]))   # [theta | pad | x | pad]
        for b in range(NB):
            for j in range(2):
                t = L.R_BLK0 + 4 * b + 2 * j
                a.linear(f"net.blocks.{b}.linear_layers.{j}", tab, (t, t + 1), H, H, Hp)
        a.linear("net.final_layer", tab, (L.R_WF, L.R_BF), 1, H, Hp)
        self.n_params = a.off
        self.index = a.index
        self.tab = tab
        self.buffers = {}

    def tc_plan(self):
        """Gather map + stage table for the wgmma evaluation path (csrc/ratio_tc.cu), or None."""
        Dt, Dx, H, NB = self.Dt, self.Dx, self.H, self.NB
        if H != 50 or Dt + Dx > 56:
            return None
        Hp, K0p, Dtp = self.Hp, self.Dtp + self.Dxp, self.Dtp
        HP8 = (H + 7) & ~7
        K0 = Dt + Dx
        k0p8 = (K0 + 7) & ~7
        t = self.tab
        w0 = int(t[L.R_W0])

        def fill0(n, k):
            col = np.where(k < Dt, k, Dtp + (k - Dt))       # packed columns [theta | pad | x | pad]
            ok = (n < H) & (k < K0)
            return np.where(ok, w0 + n * K0p + np.clip(col, 0, K0p - 1), -1)

        def hidden(woff, N, rows_valid):
            def fill(n, k):
                ok = (n < rows_valid) & (k < H)
                return np.where(ok, woff + np.minimum(n, rows_valid - 1) * Hp + np.minimum(k, H - 1), -1)
            return _tc_block(N, HP8, fill)

        stages = [(_tc_block(64, k0p8, fill0), 64, 0)]
        for b in range(NB):
            stages.append((hidden(int(t[L.R_BLK0 + 4 * b + 0]), 64, H), 64, 0))
            stages.append((hidden(int(t[L.R_BLK0 + 4 * b + 2]), 64, H), 64, 0))
        stages.append((hidden(int(t[L.R_WF]), 16, 1), 16, 0))
        return _tc_assemble([(k0p8, stages)])

    def fill_struct(self, s: "L.RatioModel", nbuf: int):
        s.Dt, s.Dx, s.H, s.NB = self.Dt, self.Dx, self.H, self.NB
        s.Dtp, s.Dxp, s.Hp = self.Dtp, self.Dxp, self.Hp
        s.rpc0, s.rpc1 = self.rpc0, self.rpc1
        s.wcap, s.nbuf, s.n_params = self.wcap, nbuf, self.n_params
        return s


@dataclass
class MlpRatioLayout(_LayoutOps):
    """Packed layout of the NRE `mlp` (NL = 2 hidden layers) and `linear` (NL = 0) classifiers
    (include/sbi_b200.h `sbi_ratio_mlp_model`), keys as in the reference's nn.Sequential
    (sbi/neural_nets/net_builders/classifier.py:49-169): `net.0/3/6.*` linears and
    `net.1/4.*` LayerNorms (absent with `norm=None`, i.e. nn.Identity), or `net.weight/bias`."""
    Dt: int
    Dx: int
    H: int = 50
    NL: int = 2
    norm: Optional[str] = "layer"
    eps: float = 1e-5
    wcap_target: int = 4096

    family = "ratio_mlp"

    def __post_init__(self):
        Dt, Dx, H, NL = self.Dt, self.Dx, self.H, self.NL
        if NL not in (0, 2) or self.norm not in ("layer", None):
            raise ValueError(f"MlpRatioLayout: NL must be 0 or 2 and norm 'layer' or None, got {NL}, {self.norm!r}")
        self.Dtp, self.Dxp, self.Hp = round4(Dt), round4(Dx), round4(H)
        K0p, Hp = self.Dtp + self.Dxp, self.Hp
        KFp = Hp if NL else K0p
        cap = max(self.wcap_target, 4 * K0p, 4 * Hp)
        (self.rpc0, self.rpc1), self.wcap = _plan_ring(cap, [(K0p, Hp), (Hp, Hp)], [4 * KFp])
        a = _Alloc()
        tab = np.zeros(10, np.int32)
        cols0 = np.concatenate([np.arange(Dt), self.Dtp + np.arange(Dx)])   # [theta | pad | x | pad]
        for l in range(NL):
            K, Kp, cols = (Dt + Dx, K0p, cols0) if l == 0 else (H, Hp, None)
            a.linear(f"net.{3 * l}", tab, (4 * l + L.RM_W0, 4 * l + L.RM_B0), H, K, Kp, cols=cols)
            if self.norm == "layer":
                o = tab[4 * l + L.RM_G0] = a.take(Hp)
                a.index[f"net.{3 * l + 1}.weight"] = o + np.arange(H)
                o = tab[4 * l + L.RM_BE0] = a.take(Hp)
                a.index[f"net.{3 * l + 1}.bias"] = o + np.arange(H)
        if NL:
            a.linear("net.6", tab, (L.RM_WF, L.RM_BF), 1, H, Hp)
        else:
            a.linear("net", tab, (L.RM_WF, L.RM_BF), 1, Dt + Dx, K0p, cols=cols0)
        self.n_params = a.off
        self.index = a.index
        self.tab = tab
        self.buffers = {}

    def fill_struct(self, s: "L.RatioMlpModel", nbuf: int):
        s.Dt, s.Dx, s.H, s.NL = self.Dt, self.Dx, self.H, self.NL
        s.Dtp, s.Dxp, s.Hp = self.Dtp, self.Dxp, self.Hp
        s.norm = L.RM_NORM_LAYER if self.norm == "layer" else L.RM_NORM_NONE
        s.ln_eps = self.eps
        s.rpc0, s.rpc1 = self.rpc0, self.rpc1
        s.wcap, s.nbuf, s.n_params = self.wcap, nbuf, self.n_params
        return s


@dataclass
class FmLayout(_LayoutOps):
    """Packed layout of the flow-matching VectorFieldMLP (include/sbi_b200.h `sbi_fm_model`), tensor
    names as in sbi/neural_nets/net_builders/vector_field_nets.py:610-719 under the
    estimator attribute `net` (FlowMatchingEstimator.net)."""
    D: int
    C: int
    H: int = 100
    NL: int = 5
    TE: int = 32
    wcap_target: int = 3200

    family = "fm"

    def __post_init__(self):
        D, C, H, NL, TE = self.D, self.C, self.H, self.NL, self.TE
        if NL < 2 or NL > 12:
            raise ValueError("2 <= num_layers <= 12")
        if TE % 2:
            raise ValueError("embedding dimension must be even")
        self.Dp, self.Cp, self.Hp, self.TEp = round4(D), round4(C), round4(H), round4(TE)
        Hp = self.Hp
        cap = max(self.wcap_target, 4 * 2 * Hp)
        (self.rpc_i, self.rpc_c, self.rpc_m, self.rpc_t, self.rpc_h, self.rpc_o), self.wcap = _plan_ring(
            cap, [(self.Dp, Hp), (self.Cp, Hp), (2 * Hp, Hp), (self.TEp, Hp), (Hp, Hp), (Hp, self.Dp)])
        a = _Alloc()
        tab = np.zeros(L.F_LAYER0 + 4 * 12, np.int32)
        a.linear("net.input_layer", tab, (L.F_WI, L.F_BI), H, D, self.Dp)
        a.linear("net.condition_layer", tab, (L.F_WC, L.F_BC), H, C, self.Cp)
        a.linear("net.input_merge_layer", tab, (L.F_WM, L.F_BM), H, 2 * H, 2 * Hp,
                 cols=np.concatenate([np.arange(H), Hp + np.arange(H)]))
        a.linear("net.time_linear_layer", tab, (L.F_WT, L.F_BT), H, TE, self.TEp)
        a.linear("net.output_layer", tab, (L.F_WO, L.F_BO), D, H, Hp)
        for i in range(NL):
            t = L.F_LAYER0 + 4 * i
            a.linear(f"net.layers.{i}", tab, (t, t + 1), H, H, Hp)
            o = tab[t + 2] = a.take(Hp)
            a.index[f"net.layers_norm.{i}.weight"] = o + np.arange(H)
            o = tab[t + 3] = a.take(Hp)
            a.index[f"net.layers_norm.{i}.bias"] = o + np.arange(H)
        self.n_params = a.off
        self.index = a.index
        self.tab = tab
        self.buffers = {}

    def fill_struct(self, s: "L.FmModel", nbuf: int):
        s.D, s.C, s.H, s.NL, s.TE = self.D, self.C, self.H, self.NL, self.TE
        s.Dp, s.Cp, s.Hp, s.TEp = self.Dp, self.Cp, self.Hp, self.TEp
        s.rpc_i, s.rpc_c, s.rpc_m = self.rpc_i, self.rpc_c, self.rpc_m
        s.rpc_t, s.rpc_h, s.rpc_o = self.rpc_t, self.rpc_h, self.rpc_o
        s.wcap, s.nbuf, s.n_params = self.wcap, nbuf, self.n_params
        s.noise_scale, s.ln_eps = 1e-3, 1e-5
        return s
