"""Estimator modules at sbi's estimator boundary, backed by the sm_90a kernels.

`NSFEstimator` mirrors `sbi.neural_nets.estimators.NFlowsFlow`
(/root/reference/sbi/neural_nets/estimators/nflows_flow.py:14-151) on the shape rules of
`ConditionalDensityEstimator` (/root/reference/sbi/neural_nets/estimators/base.py:35-306):
same method names, argument meaning, output shapes and error behaviour, and a
`state_dict()` with the reference's own keys, so reference checkpoints load verbatim.
All parameters live in ONE flat `nn.Parameter` (the packed layout of `pack.NsfLayout`);
`log_prob` is a `torch.autograd.Function` whose forward is the fused log-prob kernel and
whose backward is the fused forward+backward (VJP) kernel.  No CPU path exists.
`PackedNet` (the flat buffer and its `state_dict` mapping) and `_PackedEstimator` (statistics vector, model
struct, C entry points, scratch) are shared with the ratio and vector-field estimators.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, NamedTuple, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn

from . import _lib as L


class _Family(NamedTuple):
    """How the host hands one layout family to the library (include/sbi_b200.h)."""
    struct: type                    # the model struct of the C entry points
    tab_fields: Tuple[str, ...]     # its table pointers, in the order of `layout.tables()`
    prefix: str                     # C entry points `sbi_b200_<prefix>_<name>`
    tc: Optional[str]               # prefix of the wgmma evaluation entry points (`<tc>_tc_pack`), if any
    what: str                       # the model in error messages, formatted with the layout's fields


_FLOW = "flow (D={D}, C={C}, H={H}, num_blocks={NB})"
_CLASSIFIER = "classifier (Dt={Dt}, Dx={Dx}, H={H})"
_FAMILIES = {
    "nsf": _Family(L.NsfModel, ("d_layer_tab", "d_feat_tab"), "nsf", "nsf", _FLOW),
    # `made`: the masked residual conditioner + mixture head run on the NSF kernels (head = SBI_NSF_MOG)
    "made": _Family(L.NsfModel, ("d_layer_tab", "d_feat_tab"), "nsf", None, _FLOW),
    "maf": _Family(L.MafModel, ("d_layer_tab", "d_perm_tab"), "maf", None, _FLOW),
    "ratio": _Family(L.RatioModel, ("d_tab",), "ratio", "ratio", _CLASSIFIER),
    "ratio_mlp": _Family(L.RatioMlpModel, ("d_tab",), "ratio_mlp", None, _CLASSIFIER),
    "fm": _Family(L.FmModel, ("d_tab",), "fm", None, "vector field (D={D}, C={C}, H={H}, num_layers={NL})"),
}


class Standardize(nn.Module):
    """(t - mean) / std -- mirrors sbi.utils.sbiutils.Standardize (sbiutils.py:418-428)."""

    def __init__(self, mean, std):
        super().__init__()
        mean, std = map(torch.as_tensor, (mean, std))
        self.register_buffer("_mean", mean.clone().float())
        self.register_buffer("_std", std.clone().float())

    def forward(self, tensor):
        return (tensor - self._mean) / self._std


def _zscore_of(emb: nn.Module) -> Optional[Tuple[Tensor, Tensor]]:
    """(mean, std) of the `Standardize` in front of an embedding net, or None."""
    if isinstance(emb, nn.Sequential) and isinstance(emb[0], Standardize):
        return emb[0]._mean, emb[0]._std
    return None


class PackedNet(nn.Module):
    """Sits at `estimator.net`, where the reference keeps its network.  Owns the ONE flat fp32 parameter buffer in
    the packed layout of `layout`, the trainable mask and the layout's index tables, and maps them to and from the
    reference's `state_dict` keys (the layout's `net.` names without that prefix, then its structural `buffers`).

    buffers: {name: tensor} kept as non-persistent buffers of the net (the flows' input z-score, FM's `div_term`);
    head / tail: (reference key, buffer name) pairs saved before / after the layout's tensors and loaded back."""

    def __init__(self, layout, buffers: Optional[Dict[str, Tensor]] = None,
                 head: Sequence[Tuple[str, str]] = (), tail: Sequence[Tuple[str, str]] = ()):
        super().__init__()
        self.layout = layout
        self.flat = nn.Parameter(torch.zeros(layout.n_params, dtype=torch.float32))
        for name, t in (buffers or {}).items():
            self.register_buffer(name, t.clone().float(), persistent=False)
        self._n_tabs = 0
        for t in layout.tables():
            self.register_buffer(f"_tab{self._n_tabs}", torch.from_numpy(t.copy()), persistent=False)
            self._n_tabs += 1
        self.register_buffer("_mask", layout.trainable_mask(), persistent=False)
        # masked-out raw MADE weights, kept only so that state_dict() round-trips exactly
        self.register_buffer("_raw", torch.zeros(layout.n_params if layout._wm() else 1), persistent=False)
        self._head, self._tail = tuple(head), tuple(tail)

    def tables(self):
        """The layout's index tables on the parameter device, in `layout.tables()` order."""
        return [getattr(self, f"_tab{i}") for i in range(self._n_tabs)]

    def _raw_or_none(self):
        return self._raw if self.layout._wm() else None

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        lay = self.layout
        for key, name in self._head:
            destination[prefix + key] = getattr(self, name).detach().clone()
        for k, t in lay.unpack(self.flat, self._raw_or_none()).items():
            destination[prefix + k[len("net."):]] = t
        for k, t in lay.buffers.items():
            destination[prefix + k[len("net."):]] = t.to(self.flat.device)
        for key, name in self._tail:
            destination[prefix + key] = getattr(self, name).detach().clone()

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys,
                              unexpected_keys, error_msgs):
        lay = self.layout
        src = {}
        for k in lay.index:
            kk = prefix + k[len("net."):]
            if kk in state_dict:
                src[k] = state_dict.pop(kk)
            elif strict:
                missing_keys.append(kk)
        with torch.no_grad():
            if len(src) == len(lay.index):
                lay.pack(src, out=self.flat.data, raw_out=self._raw_or_none())
            for key, name in self._head + self._tail:
                if prefix + key in state_dict:
                    getattr(self, name).copy_(state_dict.pop(prefix + key))
            incoming = {k: state_dict.pop(prefix + k[len("net."):]) for k in list(lay.buffers)
                        if prefix + k[len("net."):] in state_dict}
            # structural buffers that are data (MAF permutations): adopt them
            if incoming and lay.load_buffers(incoming) is not None:
                for buf, t in zip(self.tables(), lay.tables()):
                    buf.copy_(torch.from_numpy(t))


class _PackedEstimator(nn.Module):
    """What the flow, ratio and vector-field estimators share: the `PackedNet` at `self.net`, the derived kernel
    inputs in `_cache` (never copied or pickled), the z-score statistics vector, the model struct of the layout's
    family, partial-gradient scratch and the wgmma operand plan.  Subclasses set `net`, `_input_shape`,
    `_condition_shape` and `_cache`, and name the sources of the statistics vector (`_stat_sources`)."""

    #: input features in front of the z-scored ones (kept at shift 0, scale 1): `made`'s dummy feature
    _STATS_OFFSET = 0
    #: whether `_stats` returns ld_zscore = sum log|input scale| (the flows' log-determinant of the z-score)
    _LD_ZSCORE = False

    input_shape = property(lambda self: self._input_shape)
    condition_shape = property(lambda self: self._condition_shape)
    layout = property(lambda self: self.net.layout)
    flat = property(lambda self: self.net.flat)
    _family = property(lambda self: _FAMILIES[self.net.layout.family])

    def __deepcopy__(self, memo):
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = {} if k == "_cache" else copy.deepcopy(v, memo)
        return new

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_cache"] = {}
        return d

    # ---- the statistics vector ------------------------------------------------------------------
    def _stat_widths(self) -> Tuple[int, int, int, int, int]:
        """(padded, real input width, padded, real condition width, trailing block length) of `_stats`."""
        lay = self.layout
        return lay.Dp, lay.D, lay.Cp, lay.C, 0

    def _stat_sources(self, raw_condition: bool):
        """((input shift, input scale) or None, (condition mean, condition std) or None, trailing block or None)."""
        raise NotImplementedError

    def _stats(self, raw_condition: bool = False) -> Tuple[Tensor, float]:
        """The kernels' statistics vector on the parameter device, `[input shift (Dp) | input scale (Dp) |
        condition mean (Cp) | condition std (Cp) | trailing block]` (include/sbi_b200.h `d_stats`; padding and
        absent statistics are 0 / 1), and ld_zscore (0 unless `_LD_ZSCORE`).  Rebuilt when a source tensor's data
        pointer or version, or the device, changes.  raw_condition: identity condition statistics, cached apart
        (see FlowEstimator.inverse_transform)."""
        inp, cond, tail = self._stat_sources(raw_condition)
        srcs = [t for t in (*(inp or ()), *(cond or ()), tail) if t is not None]
        dev = self.net.flat.device
        key = tuple((t.data_ptr(), t._version) for t in srcs) + (str(dev),)
        ck = "stats_raw" if raw_condition else "stats"
        hit = self._cache.get(ck)
        if hit is not None and hit[0] == key:
            return hit[1], hit[2]
        Dp, D, Cp, C, n_tail = self._stat_widths()
        o = self._STATS_OFFSET
        st = torch.zeros(2 * Dp + 2 * Cp + n_tail, dtype=torch.float32, device=dev)
        st[Dp:2 * Dp] = 1.0
        st[2 * Dp + Cp:2 * Dp + 2 * Cp] = 1.0
        ld = 0.0
        if inp is not None:
            st[o:D] = inp[0].reshape(-1).expand(D - o)
            st[Dp + o:Dp + D] = inp[1].reshape(-1).expand(D - o)
            if self._LD_ZSCORE:
                ld = float(torch.log(torch.abs(inp[1].double())).reshape(-1).expand(D - o).sum())
        if cond is not None:
            st[2 * Dp:2 * Dp + C] = cond[0].reshape(-1).expand(C)
            st[2 * Dp + Cp:2 * Dp + Cp + C] = cond[1].reshape(-1).expand(C)
        if tail is not None:
            st[2 * Dp + 2 * Cp:2 * Dp + 2 * Cp + tail.numel()] = tail
        self._cache[ck] = (key, st, ld)
        return st, ld

    # ---- the C entry points -----------------------------------------------------------------------
    def _model(self, nbuf: int, raw_condition: bool = False):
        """The family's model struct for the current parameters (pointers into `net` and the stats vector)."""
        net, fam = self.net, self._family
        L.require_cuda(net.flat, "estimator parameters")
        st, ld = self._stats(raw_condition)
        s = fam.struct()
        self.layout.fill_struct(s, nbuf)
        s.d_params = net.flat.data_ptr()
        for field, tab in zip(fam.tab_fields, net.tables()):
            setattr(s, field, tab.data_ptr())
        s.d_stats = st.data_ptr()
        s._keep = (st,)
        self._fill_model(s, ld)
        return s

    def _fill_model(self, s, ld: float):
        """Family-specific scalars of the model struct."""

    def _entry(self, name: str):
        """The layout's query entry point `sbi_b200_<prefix>_<name>` (one that launches nothing, e.g. `vjp_parts`)."""
        return getattr(L.load(), f"sbi_b200_{self._family.prefix}_{name}")

    def _call(self, name: str, *args):
        """`L.call` of `sbi_b200_<name>` on the parameters' device; a model that no row tile fits is named in the
        error."""
        try:
            L.call(name, *args, device=self.net.flat.device)
        except L.SbiB200Error as err:
            if err.rc != L.SBI_ESMEM:
                raise
            raise L.SbiB200Error(
                f"{name}: a row tile of this {self._family.what.format(**vars(self.layout))} needs more than "
                "the 227 KB of shared memory one CTA can use on sm_90a (SBI_ESMEM)", err.rc) from None

    def _gpart(self, n_part: int) -> Tensor:
        """Partial-gradient scratch, (>= n_part, n_params), zeroed when (re)allocated."""
        buf = self._cache.get("gpart")
        dev = self.net.flat.device
        if buf is None or buf.shape[0] < n_part or buf.device != dev:
            buf = torch.zeros(max(n_part, 1), self.layout.n_params, dtype=torch.float32, device=dev)
            self._cache["gpart"] = buf
        return buf

    def _tc_state(self, m):
        """`NsfTc` descriptor of the family's wgmma evaluation kernel for the current parameters, or None if the
        family has none, SBI_B200_TC=0, or the model is outside what the kernel instantiates.  The operands are
        re-packed from the flat parameter buffer on every call (a ~1 MB elementwise kernel): the optimizer
        kernels update the parameters through raw pointers, so no version counter could be trusted."""
        tc = self._family.tc
        if tc is None or os.environ.get("SBI_B200_TC", "") == "0":
            return None
        dev = self.net.flat.device
        st = self._cache.get("tc")
        if st is None or st["dev"] != dev:
            plan = self.layout.tc_plan()
            st = {"dev": dev, "plan": plan}
            if plan is not None:
                st.update(src=torch.as_tensor(plan["src"], device=dev), tab=torch.as_tensor(plan["tab"], device=dev),
                          tcw=torch.empty(plan["n_words"], dtype=torch.float32, device=dev))
            self._cache["tc"] = st
        if st["plan"] is None:
            return None
        desc = L.NsfTc(st["plan"]["n_words"], st["plan"]["stage_cap"], st["src"].data_ptr(),
                       st["tab"].data_ptr(), st["tcw"].data_ptr())
        if not getattr(L.load(), f"sbi_b200_{tc}_tc_supported")(C.byref(m), C.byref(desc)):
            return None
        self._call(f"{tc}_tc_pack", m, desc)
        return desc


class FlowEstimator(_PackedEstimator):
    r"""Normalizing flow q(input | condition) evaluated by hand-written sm_90a kernels
    (families: neural spline flow `nsf`, masked autoregressive flow `maf`)."""

    _LD_ZSCORE = True

    def __init__(self, layout, input_shape, condition_shape, shift: Tensor,
                 scale: Tensor, cond_mean: Optional[Tensor], cond_std: Optional[Tensor],
                 embedding_net: Optional[nn.Module] = None):
        super().__init__()
        self._input_shape = torch.Size(input_shape)
        self._condition_shape = torch.Size(condition_shape)
        user_net = embedding_net if embedding_net is not None else nn.Identity()
        self._embed_identity = isinstance(user_net, nn.Identity)
        if cond_mean is not None:
            emb = nn.Sequential(Standardize(cond_mean, cond_std), user_net)
        else:
            emb = user_net
        zscore = [("_transform._transforms.0._shift", "_shift"), ("_transform._transforms.0._scale", "_scale")]
        # plays the role of the nflows `Flow` object that sits at `estimator.net`
        self.net = PackedNet(layout, dict(_shift=shift, _scale=scale), head=zscore if layout.zscore_input else ())
        self.net._embedding_net = emb
        self._cache = {}

    @property
    def embedding_net(self) -> nn.Module:
        return self.net._embedding_net

    # ---- kernel-side views --------------------------------------------------------------------
    def _stat_sources(self, raw_condition: bool):
        net = self.net
        cond = None if raw_condition or not self._embed_identity else _zscore_of(net._embedding_net)
        return (net._shift, net._scale), cond, None

    def _fill_model(self, s, ld: float):
        s.ld_zscore = ld

    def _embed(self, condition: Tensor) -> Tensor:
        """Context fed to the kernels.  Identity embedding: raw condition (standardised
        in-kernel); otherwise the torch embedding net runs first."""
        if self._embed_identity:
            return condition.reshape(condition.shape[0], -1)
        return self.net._embedding_net(condition).reshape(condition.shape[0], -1)

    # ---- shape handling: base.py:84-198 --------------------------------------------------------
    def _check_condition_shape(self, condition: Tensor):
        exp = self.condition_shape
        if len(condition.shape) < len(exp):
            raise ValueError(
                "Dimensionality of condition is too small and does not match the "
                f"expected dimensionality {len(exp)}. It should "
                f"be compatible with condition_shape {exp}.")
        if condition.shape[-len(exp):] != exp:
            raise ValueError(
                f"Shape of condition {condition.shape[-len(exp):]} does not match the "
                f"expected input dimensionality {exp}, as "
                "provided by condition_shape. Please reshape it accordingly.")

    def _check_input_shape(self, input: Tensor):
        exp = self.input_shape
        if len(input.shape) < len(exp):
            raise ValueError(
                "Dimensionality of input is too small and does not match the "
                f"expected dimensionality {len(exp)}. It should "
                f"be compatible with the provided input_shape {exp}.")
        if input.shape[-len(exp):] != exp:
            raise ValueError(
                f"Shape of input {input.shape[-len(exp):]} does not match the "
                f"expected input dimensionality {exp}, as "
                "provided by input_shape. Please reshape it accordingly.")

    def _align(self, input: Tensor, condition: Tensor):
        """_broadcast_and_align (base.py:142-198) without materialising a broadcast
        condition: returns input (S*B, D), condition rows and a `shared` flag."""
        in_ev, c_ev = len(self.input_shape), len(self.condition_shape)
        if input.dim() <= in_ev + 1:
            input = input.unsqueeze(0)
        S, Bi = input.shape[0], input.shape[1]
        cond_has_sample = condition.dim() > c_ev + 1
        Bc = condition.shape[1] if cond_has_sample else condition.shape[0]
        try:
            B = torch.broadcast_shapes((Bi,), (Bc,))[0]
        except RuntimeError as err:
            raise RuntimeError(
                "Expected `input` and `condition` to have broadcastable batch "
                "dimensions: their batch sizes must match, or one of them must be 1. "
                f"Got input={Bi} and condition={Bc}.") from err
        input = input.expand(S, B, *self.input_shape).reshape(S * B, -1)
        if not cond_has_sample and Bc == 1:
            return input, condition.reshape(1, *self.condition_shape), True, S, B
        if cond_has_sample:
            condition = condition.expand(S, B, *self.condition_shape)
        else:
            condition = condition.expand(B, *self.condition_shape).unsqueeze(0).expand(
                S, B, *self.condition_shape)
        return input, condition.reshape(S * B, *self.condition_shape), False, S, B

    # ---- the reference API ------------------------------------------------------------------------
    def log_prob(self, input: Tensor, condition: Tensor) -> Tensor:
        """(sample_dim, batch_dim) log-probabilities; nflows_flow.py:77-97."""
        self._check_input_shape(input)
        self._check_condition_shape(condition)
        if not self.net.flat.is_cuda:
            # the reference probes a freshly built (CPU-resident) net with two CPU rows before it
            # moves it to the training device (user_input_checks.py:767-795): device hop, no CPU math
            from ._refabc import hop_to_device
            return hop_to_device(self, "log_prob", input, condition)
        inp, cond, shared, S, B = self._align(input, condition)
        ctx = self._embed(cond)
        lp = _NsfLogProb.apply(self.net.flat, inp.contiguous().float(), ctx.contiguous().float(),
                               self, shared)
        return lp.reshape(S, B)

    def loss(self, input: Tensor, condition: Tensor) -> Tensor:
        """(batch_dim,) negative log-probabilities; nflows_flow.py:99-109."""
        return -self.log_prob(input.unsqueeze(0), condition)[0]

    def inverse_transform(self, input: Tensor, condition: Tensor) -> Tensor:
        """Base-space noise of the inputs; nflows_flow.py:42-75.  Like the reference (:73), the
        RAW condition feeds the transform here: neither the condition z-scoring nor the
        embedding net is applied on this code path."""
        self._check_condition_shape(condition)
        cdims = len(self.condition_shape)
        bshape = torch.broadcast_shapes(input.shape[:-1], condition.shape[:-cdims])
        inp = input.expand(bshape + (input.shape[-1],)).reshape(-1, input.shape[-1])
        cond = condition.expand(bshape + self.condition_shape).reshape(-1, *self.condition_shape)
        ctx = cond.reshape(cond.shape[0], -1)
        if ctx.shape[1] != self.layout.C:
            raise ValueError("inverse_transform: the raw condition does not have the embedded "
                             "context size (reference behaviour: no embedding on this path)")
        _, noise = self._logprob_raw(inp.contiguous().float(), ctx.contiguous().float(), False,
                                     want_noise=True, raw_condition=True)
        return noise.reshape(bshape + (noise.shape[-1],))

    @torch.no_grad()
    def sample(self, sample_shape, condition: Tensor) -> Tensor:
        """(*sample_shape, batch_dim, *input_shape); nflows_flow.py:111-128.  Noise is drawn
        with torch.randn on the parameter device in the order nflows draws it
        (B*n rows, condition-major), then pushed through the inverse-flow kernel."""
        self._check_condition_shape(condition)
        Bc = condition.shape[0]
        n = torch.Size(sample_shape).numel()
        D = self.layout.D
        noise = torch.randn(Bc * n, D, device=self.net.flat.device)
        x, _ = self.inverse_flow(noise, condition, n)
        x = x.reshape(Bc, n, D).transpose(0, 1)
        return x.reshape((*sample_shape, Bc, *self.input_shape))

    @torch.no_grad()
    def sample_and_log_prob(self, sample_shape, condition: Tensor, **kwargs):
        """nflows_flow.py:130-151 (via nflows Flow.sample_and_log_prob)."""
        Bc = condition.shape[0]
        n = torch.Size(sample_shape).numel()
        D = self.layout.D
        noise = torch.randn(Bc * n, D, device=self.net.flat.device)
        base_lp = -0.5 * (noise ** 2).sum(1) - 0.5 * D * 1.8378770664093453
        x, lad = self.inverse_flow(noise, condition, n)
        samples = x.reshape(Bc, n, D).reshape((*sample_shape, Bc, -1))
        log_probs = (base_lp - lad).reshape(Bc, n).reshape((*sample_shape, -1))
        return samples, log_probs

    @torch.no_grad()
    def inverse_flow(self, noise: Tensor, condition: Tensor, reps: int = 1):
        """x = T^{-1}(noise | condition); `noise` (B*reps, D) condition-major,
        `condition` (B, *condition_shape).  Returns (x, log|det dx/dnoise|)."""
        L.require_cuda(noise, "noise")
        Bc = condition.shape[0]
        ctx = self._embed(condition.to(noise.device)).contiguous().float()
        shared = Bc == 1
        if not shared:
            ctx = ctx.repeat_interleave(reps, dim=0).contiguous()
        noise = noise.contiguous().float()
        R = noise.shape[0]
        out = torch.empty_like(noise)
        lad = torch.empty(R, dtype=torch.float32, device=noise.device)
        m = self._model(nbuf=2)
        rows = L.rows(noise, ctx, shared=shared)
        if R >= self.TC_MIN_ROWS or os.environ.get("SBI_B200_TC", "") == "1":
            tc = self._tc_state(m)
            if tc is not None:
                self._call("nsf_inverse_tc", m, tc, rows, out, lad)
                return out, lad
        self._call(f"{self._family.prefix}_inverse", m, rows, out, lad)
        return out, lad

    # ---- tensor-core bulk path (nsf only) --------------------------------------------------------
    #: rows from which log_prob / sampling go through the wgmma kernel (csrc/nsf_tc.cu).  The
    #: crossover against the SIMT kernel has not been measured for the wgmma kernel (profiles/tc_cross.py
    #: measures it); 1024 is carried over from the earlier tensor-core design.
    #: SBI_B200_TC=0 disables, =1 forces (`_PackedEstimator._tc_state`).
    TC_MIN_ROWS = int(os.environ.get("SBI_B200_TC_MIN_ROWS", 1024))

    # ---- fused forward+backward of a batch (parameter / input / condition gradients) --------------
    #: rows from which the training VJP runs on the tensor cores (csrc/nsf_vjp_tc.cu) when only parameter
    #: gradients are wanted (threshold not measured for the wgmma kernels; profiles/vjp_cross.py measures
    #: it); SBI_B200_VJP_TC=0 disables, =1 forces
    VJP_TC_MIN_ROWS = int(os.environ.get("SBI_B200_VJP_TC_MIN_ROWS", 256))

    def _tc_train_state(self, m, pack: bool = True):
        """(tc_fwd, tc_bwd, tc_both) operand descriptors for the tensor-core training step, freshly
        packed from the current parameters by ONE pack launch over both plans (`tc_both`), or None."""
        if self.layout.family != "nsf" or os.environ.get("SBI_B200_VJP_TC", "") == "0":
            return None
        flat = self.net.flat
        st = self._cache.get("tc_train")
        if st is None or st["dev"] != flat.device:
            pf, pb = self.layout.tc_plan(), self.layout.tc_bwd_plan()
            st = {"dev": flat.device, "ok": pf is not None and pb is not None}
            if st["ok"]:
                import numpy as np
                dev = flat.device
                st.update(nf=pf["n_words"], nb=pb["n_words"], cap_f=pf["stage_cap"], cap_b=pb["stage_cap"],
                          src=torch.as_tensor(np.concatenate([pf["src"], pb["src"]]), device=dev),
                          tab_f=torch.as_tensor(pf["tab"], device=dev), tab_b=torch.as_tensor(pb["tab"], device=dev),
                          tcw=torch.empty(pf["n_words"] + pb["n_words"], dtype=torch.float32, device=dev))
            self._cache["tc_train"] = st
        if not st["ok"]:
            return None
        both = L.NsfTc(st["nf"] + st["nb"], st["cap_f"], st["src"].data_ptr(), st["tab_f"].data_ptr(),
                       st["tcw"].data_ptr())
        tcf = L.NsfTc(st["nf"], st["cap_f"], st["src"].data_ptr(), st["tab_f"].data_ptr(), st["tcw"].data_ptr())
        tcb = L.NsfTc(st["nb"], st["cap_b"], st["src"].data_ptr() + 4 * st["nf"], st["tab_b"].data_ptr(),
                      st["tcw"].data_ptr() + 4 * st["nf"])
        if not L.load().sbi_b200_nsf_vjp_tc_supported(C.byref(m), C.byref(tcf), C.byref(tcb)):
            st["ok"] = False
            return None
        if pack:
            self._call("nsf_tc_pack", m, both)
        return tcf, tcb, both

    def vjp_parts(self, R: int, param_grads_only: bool = True) -> int:
        """Number of partial-gradient slabs `vjp` writes for R rows."""
        if self._vjp_uses_tc(R, param_grads_only):
            return L.load().sbi_b200_nsf_vjp_tc_parts(R)
        return self._entry("vjp_parts")(R)

    def _vjp_uses_tc(self, R: int, param_grads_only: bool) -> bool:
        env = os.environ.get("SBI_B200_VJP_TC", "")
        if self.layout.family != "nsf" or env == "0" or not param_grads_only:
            return False
        if R < self.VJP_TC_MIN_ROWS and env != "1":
            return False
        st = self._cache.get("tc_train")
        if st is not None and st["dev"] == self.net.flat.device:
            return bool(st["ok"])
        return self._tc_train_state(self._model(nbuf=3)) is not None

    def vjp_cond_uses_tc(self, R: int) -> bool:
        """Whether the trainer's step with a condition gradient (embedding net) runs on the tensor cores
        (`sbi_b200_nsf_vjp_tc_cond`): that instantiation adds no shared memory, so it runs wherever the
        parameter-only step does.  `log_prob().backward()` does not use this path."""
        return self._vjp_uses_tc(R, True)

    def _vjp_save(self, nbytes: int):
        """(pointer, bytes) of the VJP kernels' activation scratch, grown to at least `nbytes` bytes on the
        parameter device, or (None, 0) when `nbytes` is 0 (the kernel keeps nothing)."""
        if nbytes == 0:
            return None, 0
        dev = self.net.flat.device
        save = self._cache.get("vjp_save")
        if save is None or save.numel() * 4 < nbytes or save.device != dev:
            save = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=dev)
            self._cache["vjp_save"] = save
        return save.data_ptr(), save.numel() * 4

    def vjp(self, m, rows, R: int, gout, g_const: float, logp, gpart, ginput=None, gcond=None, loss_acc=None,
            cond_tc: bool = False):
        """One launch (pair) of the fused forward+backward of `R` rows: partial parameter gradients of
        sum_r g_r log q_r into `gpart` ((vjp_parts(R, ...), n_params)), optionally the gradients
        w.r.t. the inputs / conditions, the log-probs and the loss statistics.  Tensor-core kernels when
        only parameter gradients are wanted, or with `cond_tc` (the trainer's step with an embedding net, after
        `vjp_cond_uses_tc(R)`) parameter and condition gradients; else the SIMT kernel."""
        lib = L.load()
        if ginput is None and (gcond is None or cond_tc) and self._vjp_uses_tc(R, True):
            tcs = self._tc_train_state(m)
            if tcs is not None:
                save, nbytes = self._vjp_save(lib.sbi_b200_nsf_vjp_tc_save_bytes(C.byref(m), R))
                if gcond is not None:
                    self._call("nsf_vjp_tc_cond", m, tcs[0], tcs[1], rows, gout, g_const, logp, gpart, loss_acc, gcond,
                               save, nbytes)
                    return
                self._call("nsf_vjp_tc", m, tcs[0], tcs[1], rows, gout, g_const, logp, gpart, loss_acc, save, nbytes)
                return
        prefix = self._family.prefix
        args = (m, rows, gout, g_const, logp, gpart, ginput, gcond, loss_acc)
        if prefix == "nsf":       # `nsf` and `made`: the SIMT kernel spills its activations
            args += self._vjp_save(lib.sbi_b200_nsf_vjp_save_bytes(C.byref(m), R))
        self._call(f"{prefix}_vjp", *args)

    # ---- raw kernel entry (no autograd) --------------------------------------------------------------
    def _logprob_raw(self, inp: Tensor, ctx: Tensor, shared: bool, want_noise=False,
                     index: Optional[Tensor] = None, n_rows: Optional[int] = None,
                     raw_condition: bool = False, out: Optional[Tensor] = None):
        """Log-probs (and with `want_noise` the base-space noise) of R rows, R = n_rows or len(inp), with the
        condition of row r at ctx[r] (ctx[0] when `shared`) and optional row `index`; written into `out` (R,) if
        given.  wgmma kernel from TC_MIN_ROWS rows when the model fits it, else the SIMT kernel."""
        L.require_cuda(inp, "input")
        L.require_cuda(ctx, "condition")
        R = inp.shape[0] if n_rows is None else n_rows
        lp = torch.empty(R, dtype=torch.float32, device=inp.device) if out is None else out
        noise = torch.empty(R, self.layout.D, dtype=torch.float32, device=inp.device) if want_noise else None
        m = self._model(nbuf=2, raw_condition=raw_condition)
        rows = L.rows(inp, ctx, index, R, shared)
        if R >= self.TC_MIN_ROWS or os.environ.get("SBI_B200_TC", "") == "1":
            tc = self._tc_state(m)
            if tc is not None:
                self._call("nsf_logprob_tc", m, tc, rows, lp, noise)
                return lp, noise
        self._call(f"{self._family.prefix}_logprob", m, rows, lp, noise)
        return lp, noise


class _NsfLogProb(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flat, inp, cond, est, shared: bool):
        lp, _ = est._logprob_raw(inp, cond, shared)
        ctx.save_for_backward(inp, cond)
        ctx.est, ctx.shared = est, shared
        return lp

    @staticmethod
    def backward(ctx, g):
        inp, cond = ctx.saved_tensors
        est, shared = ctx.est, ctx.shared
        need_flat, need_inp, need_cond = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        R = inp.shape[0]
        n_part = est.vjp_parts(R, not (need_inp or need_cond))
        gpart = est._gpart(n_part)
        ginp = torch.empty_like(inp) if need_inp else None
        gcond = torch.empty(R, cond.shape[1], dtype=torch.float32, device=inp.device) if need_cond else None
        m = est._model(nbuf=3)
        rows = L.rows(inp, cond, shared=shared)
        g = g.contiguous().float()
        est.vjp(m, rows, R, g, 0.0, None, gpart, ginp, gcond, None)
        gflat = L.reduce_partials(gpart, n_part, est.layout.n_params) if need_flat else None
        if need_cond and shared:
            gcond = gcond.sum(0, keepdim=True)
        return gflat, ginp, gcond, None, None


NSFEstimator = FlowEstimator
MAFEstimator = FlowEstimator


class MadeEstimator(FlowEstimator):
    r"""sbi's `made` density estimator (flow.py:37-112): z-scoring followed by a conditional MADE with a
    mixture-of-Gaussians head (nflows MADEMoG behind sbi's MADEMoGWrapper, nn_utils.py:133-201), evaluated by
    the NSF kernels with head = SBI_NSF_MOG.  The wrapper's dummy first feature is part of the network: the
    kernels see `input dim + 1` features, feature 0 is fed 0 by `log_prob` and -- like the reference's
    `_sample` -- drawn from its own mixture in `sample` and dropped from the result."""

    _STATS_OFFSET = 1        # feature 0 (dummy): shift 0, scale 1

    @staticmethod
    def with_dummy(inp: Tensor) -> Tensor:
        """(R, D) -> (R, D + 1) with the wrapper's zero first feature (nn_utils.py:166-167)."""
        return torch.cat([torch.zeros(inp.shape[0], 1, dtype=inp.dtype, device=inp.device), inp], dim=1)

    def log_prob(self, input: Tensor, condition: Tensor) -> Tensor:
        self._check_input_shape(input)
        self._check_condition_shape(condition)
        if not self.net.flat.is_cuda:
            from ._refabc import hop_to_device
            return hop_to_device(self, "log_prob", input, condition)
        inp, cond, shared, S, B = self._align(input, condition)
        ctx = self._embed(cond)
        lp = _NsfLogProb.apply(self.net.flat, self.with_dummy(inp.float()).contiguous(), ctx.contiguous().float(),
                               self, shared)
        return lp.reshape(S, B)

    def inverse_transform(self, input: Tensor, condition: Tensor) -> Tensor:
        """The flow's transform is the z-scoring alone (CompositeTransform([standardize, identity]))."""
        return input * self.net._scale + self.net._shift

    @torch.no_grad()
    def sample(self, sample_shape, condition: Tensor) -> Tensor:
        """(*sample_shape, batch_dim, *input_shape): D + 1 sequential conditioner passes in one kernel
        (csrc/nsf.cu `made_sample_kernel`); the normal draws and the component-selecting uniforms come from
        torch on the parameter device, condition-major like nflows (`repeat_interleave(context, n)`)."""
        self._check_condition_shape(condition)
        dev = self.net.flat.device
        Bc = condition.shape[0]
        n = torch.Size(sample_shape).numel()
        Dn = self.layout.D
        R = Bc * n
        noise = torch.randn(R, Dn, device=dev)
        unif = torch.rand(R, Dn, device=dev)
        ctx = self._embed(condition.to(dev)).contiguous().float()
        shared = Bc == 1
        if not shared:
            ctx = ctx.repeat_interleave(n, dim=0).contiguous()
        out = torch.empty(R, Dn, dtype=torch.float32, device=dev)
        m = self._model(nbuf=2)
        self._call("made_sample", m, L.rows(noise, ctx, shared=shared), unif, out)
        x = out[:, 1:].reshape(Bc, n, Dn - 1).transpose(0, 1)
        return x.reshape((*sample_shape, Bc, *self.input_shape))

    @torch.no_grad()
    def sample_and_log_prob(self, sample_shape, condition: Tensor, **kwargs):
        samples = self.sample(sample_shape, condition)
        n = torch.Size(sample_shape).numel()
        flat = samples.reshape(n, condition.shape[0], -1)
        return samples, self.log_prob(flat, condition).reshape((*sample_shape, -1))

    def inverse_flow(self, noise: Tensor, condition: Tensor, reps: int = 1):
        raise NotImplementedError("`made` is a conditional distribution, not an invertible flow of base noise")
