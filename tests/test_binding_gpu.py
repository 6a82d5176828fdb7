"""Every kernel launch goes on torch's current stream of the device its tensors live on, whatever stream or
device is current: with a side stream current, while a sampler captures its CUDA graph, and with the work on
cuda:1 while cuda:0 is current.  The loaded library is wrapped so that every entry point that takes a stream
records the handle it received next to the current stream of the work's device at that moment, then calls
through; the results must equal those of a run on the default stream of the work's device."""
import ctypes as C

import numpy as np
import pytest
import torch

from sbi_b200 import _lib
from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu


class _Recorder:
    """Stands in for the object `_lib.load()` returns."""

    def __init__(self, lib):
        self.device = None
        self.log = []           # (entry point, stream handle received, current stream of `device`)
        for name, (_, argtypes) in _lib._EXPORTS.items():
            fn = getattr(lib, name)
            setattr(self, name, self._wrap(name, fn) if argtypes and argtypes[-1] is _lib._Stream else fn)

    def _wrap(self, name, fn):
        def launch(*args):
            s = args[-1].value if isinstance(args[-1], C.c_void_p) else args[-1]
            self.log.append((name[len("sbi_b200_"):], s or 0, torch.cuda.current_stream(self.device).cuda_stream))
            return fn(*args)
        return launch


@pytest.fixture
def recorder(cuda_lib, monkeypatch):
    rec = _Recorder(cuda_lib)
    monkeypatch.setattr(_lib, "_lib", rec)
    return rec


def _normal(p):
    return -0.5 * (p * p).sum(-1)


def _proposal(dev):
    return torch.distributions.MultivariateNormal(torch.zeros(2, device=dev), 4.0 * torch.eye(2, device=dev))


def _nsf(dev):
    flow, theta, x = oracle_nsf(10, 10, n=2500)
    est = b200_from_oracle(flow, theta, x, device=dev)
    inp, cond = theta[:64].to(dev).requires_grad_(True), x[:64].to(dev)
    out = [est.log_prob(inp, cond)[0]]                                  # SIMT forward, input + parameter VJP
    out[0].sum().backward()
    out += [inp.grad, est.flat.grad.clone()]
    est.zero_grad()
    with torch.no_grad():
        out.append(est.log_prob(theta[:2048].to(dev), x[:2048].to(dev))[0])      # tensor-core forward
    est.loss(theta[:1024].to(dev), x[:1024].to(dev)).mean().backward()          # tensor-core training pair
    out += [est.flat.grad, est.sample((64,), x[:1].to(dev)), est.sample((2048,), x[1:2].to(dev))]
    return out


def _ratio(dev):
    from sbi_b200.ratio import build_resnet_classifier
    g = torch.Generator().manual_seed(0)
    theta, x = torch.randn(300, 4, generator=g), torch.randn(300, 6, generator=g)
    est = build_resnet_classifier(theta, x).to(dev)
    th = theta[:100].to(dev).requires_grad_(True)
    logits = est(th, x[:100].to(dev))
    logits.sum().backward()
    return [logits, th.grad, est.net.flat.grad]


def _fm_estimator(dev):
    from sbi_b200.flowmatching import posterior_flow_nn
    g = torch.Generator().manual_seed(0)
    theta, x = torch.randn(300, 3, generator=g), torch.randn(300, 5, generator=g)
    return posterior_flow_nn("mlp")(theta, x).to(dev), theta.to(dev), x.to(dev)


def _fm(dev):
    est, theta, x = _fm_estimator(dev)
    t = torch.full((64,), 0.3, device=dev)
    with torch.no_grad():
        out = [est(theta[:64], x[:64], t), *est.forward_and_divergence(theta[:64], x[:64], t)]
    est.loss(theta[:64], x[:64]).mean().backward()
    return out + [est.net.flat.grad]


def _ode_sde(dev):
    from sbi_b200.flowmatching import sample_ode, sample_sde
    est, _, x = _fm_estimator(dev)
    return [sample_ode(est, 64, x[:1]), sample_sde(est, 64, x[:1], steps=20)]


def _slice(dev):
    from sbi_b200.samplers import SliceSamplerVectorized
    s = SliceSamplerVectorized(_normal, np.full((8, 2), 0.1), num_chains=8, seed=3, check_every=4, graph=True,
                               device=str(dev))
    return [s.run(40)]


def _hmc(dev):
    from sbi_b200.hmc import HMCSamplerVectorized
    s = HMCSamplerVectorized(_normal, np.full((4, 2), 0.1), num_chains=4, warmup_steps=8, check_every=4, graph=True,
                             device=str(dev))
    return [s.run(8)]


def _rejection(dev):
    from sbi_b200.samplers import rejection_sample
    samples, _ = rejection_sample(_normal, _proposal(dev), num_samples=64, num_samples_to_find_max=64,
                                  num_iter_to_find_max=3, device=str(dev))
    return [samples]


def _sir(dev):
    from sbi_b200.samplers import sampling_importance_resampling
    return [sampling_importance_resampling(_normal, _proposal(dev), num_samples=32, num_candidate_samples=8,
                                           device=str(dev))]


def _mmd(dev):
    from sbi_b200.misspecification import compute_rbf_mmd, rbf_kernel
    g = torch.Generator().manual_seed(0)
    x, y = torch.randn(50, 3, generator=g).to(dev), torch.randn(40, 3, generator=g).to(dev)
    return [compute_rbf_mmd(x, y, 1.5), rbf_kernel(x, y, 1.5)]


def _lc2st(dev):
    from sbi_b200.lc2st import LC2ST
    g = torch.Generator().manual_seed(0)
    theta, x = torch.randn(200, 2, generator=g), torch.randn(200, 2, generator=g)
    post = x + 0.5 * torch.randn(200, 2, generator=g)
    lc = LC2ST(theta, x, post, num_trials_null=2, classifier_kwargs=dict(max_iter=5), device=str(dev))
    lc.train_on_observed_data(seed=0)
    return [*lc.trained_clfs[0].coefs_, np.float64(lc.get_statistic_on_observed_data(post[:50], x[0]))]


def _npe(dev):
    from sbi_b200.inference import NPE
    g = torch.Generator().manual_seed(0)
    theta = torch.randn(1000, 3, generator=g)
    x = theta + 0.3 * torch.randn(1000, 3, generator=g)
    prior = torch.distributions.MultivariateNormal(torch.zeros(3), torch.eye(3))
    net = NPE(prior, device=str(dev)).append_simulations(theta, x).train(max_num_epochs=2, training_batch_size=100)
    return [net.flat.detach()]


# workload: (its run, entry points it must launch)
WORKLOADS = {
    "nsf": (_nsf, {"nsf_logprob", "nsf_vjp", "nsf_logprob_tc", "nsf_tc_pack", "nsf_vjp_tc", "nsf_inverse",
                   "nsf_inverse_tc", "reduce_partials"}),
    "ratio": (_ratio, {"ratio_forward", "ratio_vjp_inputs", "reduce_partials"}),
    "fm": (_fm, {"fm_forward", "fm_forward_div", "fm_loss_vjp", "fm_loss_vjp_cond", "reduce_partials"}),
    "ode_sde": (_ode_sde, {"ode_stage", "ode_error_commit", "fm_forward", "sde_em_step"}),
    "slice": (_slice, {"slice_init", "slice_step"}),
    "hmc": (_hmc, {"hmc_init", "hmc_step"}),
    "rejection": (_rejection, {"reject_compact"}),
    "sir": (_sir, {"sir_select"}),
    "mmd": (_mmd, {"mmd", "rbf_matrix"}),
    "lc2st": (_lc2st, {"lc2st_train", "lc2st_eval"}),
}
NPE_WORKLOAD = (_npe, {"reduce_partials_norm", "adam_clip_step_norm", "nll_stats"})


def _run(run, dev):
    torch.manual_seed(0)
    out = run(dev)
    torch.cuda.synchronize(dev)
    return [t.detach().cpu() if isinstance(t, torch.Tensor) else np.asarray(t) for t in out]


def _assert_equal(got, want, tag):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        same = torch.equal(a, b) if isinstance(a, torch.Tensor) else np.array_equal(a, b)
        assert same, f"{tag}: output {i} differs from the run on the default stream"


def _assert_launches(log, must, not_streams=()):
    assert must <= {name for name, _, _ in log}, sorted(must - {name for name, _, _ in log})
    for name, got, current in log:
        assert got == current, f"{name} launched on stream {got:#x}, the current stream is {current:#x}"
        assert got != 0 and got not in not_streams, f"{name} launched on stream {got:#x}"


@pytest.mark.parametrize("workload", list(WORKLOADS))
def test_launches_go_on_the_current_stream(recorder, workload):
    run, must = WORKLOADS[workload]
    dev = torch.device("cuda", torch.cuda.current_device())
    recorder.device = dev
    want = _run(run, dev)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    recorder.log.clear()
    with torch.cuda.stream(side):
        got = _run(run, dev)
    _assert_launches(recorder.log, must)
    _assert_equal(got, want, workload)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("workload", list(WORKLOADS) + ["npe"])
def test_launches_follow_the_tensors_device(recorder, workload):
    """cuda:0 stays current, with a side stream of its own, while the work runs on cuda:1 tensors."""
    run, must = NPE_WORKLOAD if workload == "npe" else WORKLOADS[workload]
    d0, d1 = torch.device("cuda", 0), torch.device("cuda", 1)
    recorder.device = d1
    with torch.cuda.device(d1):
        want = _run(run, d1)
    s0, s1 = torch.cuda.Stream(device=d0), torch.cuda.Stream(device=d1)
    s1.wait_stream(torch.cuda.current_stream(d1))
    prev1 = torch.cuda.current_stream(d1)
    with torch.cuda.device(d1):
        torch.cuda.set_stream(s1)          # cuda:1's current stream; cuda:0 becomes current again below
    recorder.log.clear()
    try:
        with torch.cuda.device(d0), torch.cuda.stream(s0):
            assert torch.cuda.current_device() == 0
            got = _run(run, d1)
    finally:
        with torch.cuda.device(d1):
            torch.cuda.set_stream(prev1)
    _assert_launches(recorder.log, must, not_streams=(s0.cuda_stream,))
    _assert_equal(got, want, workload)
