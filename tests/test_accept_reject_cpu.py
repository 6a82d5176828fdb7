"""`posteriors.accept_reject_sample`, the one accept/reject loop of the direct and vector-field posteriors and of
`RestrictedPrior`, on the CPU: against the UNMODIFIED reference's `accept_reject_sample` (rejection.py:230-457,
through oracle.ref_shim) with a seeded fake proposal for one observation, and against its own definition for
several observations and after a timeout."""
import logging
import re
import time

import pytest
import torch

from oracle import ref_shim
from sbi_b200.posteriors import accept_reject_sample

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")


@pytest.fixture(scope="module")
def ref_loop():
    assert ref_shim.install()
    from sbi.samplers.rejection.rejection import accept_reject_sample as ref
    return ref


class Proposal:
    """Uniform draws in [0, 1) of shape (n, *batch, 2) from its own generator; records every batch it returns."""

    def __init__(self, batch=(1,), seed=0, delay=0.0):
        self.batch, self.delay = batch, delay
        self.g = torch.Generator().manual_seed(seed)
        self.draws = []

    def __call__(self, shape, **kw):
        time.sleep(self.delay)
        d = torch.rand(torch.Size(shape).numel(), *self.batch, 2, generator=self.g)
        self.draws.append(d)
        return d

    @property
    def sizes(self):
        return [d.shape[0] for d in self.draws]


class Scripted:
    """Accepts `th[..., 0] < p` with one threshold per round (the last repeats): 0 rejects all, 1 accepts all."""

    def __init__(self, *p):
        self.p, self.calls = p, 0

    def __call__(self, th):
        p = self.p[min(self.calls, len(self.p) - 1)]
        self.calls += 1
        return (th[..., 0] < p).reshape(-1)


def _both(ref_loop, accept, caplog, **kw):
    """Runs the reference's loop and ours from the same proposal seed: (samples, rate, batch sizes, log) each."""
    out = []
    for loop in (ref_loop, accept_reject_sample):
        prop = Proposal()
        caplog.clear()
        with caplog.at_level(logging.WARNING):
            s, r = loop(prop, Scripted(*accept), **kw)
        out.append((s, r, prop.sizes, caplog.text))
    return out


@needs_ref
@pytest.mark.parametrize("accept, num_samples, max_batch", [
    ((0.5,), 1000, 400),                  # many rounds at about 50 %
    ((0.0, 0.02, 1.0), 300, 1000),        # nothing, then 2 %, then everything: the last round overshoots
    ((1.0,), 250, 10_000),                # everything in the first round
    ((0.0, 0.0, 0.3), 120, 500),          # two empty rounds
])
def test_one_observation_bit_equal_to_reference(ref_loop, caplog, accept, num_samples, max_batch):
    (rs, rr, rsz, rlog), (s, r, sz, log) = _both(ref_loop, accept, caplog, num_samples=num_samples,
                                                 max_sampling_batch_size=max_batch)
    assert sz == rsz and sz[0] == min(num_samples, max_batch)
    assert s.shape == rs.shape == (num_samples, 1, 2) and torch.equal(s, rs)
    assert r.dtype == rr.dtype == torch.float32 and torch.equal(r, rr)
    assert (log == "") == (rlog == "")


@needs_ref
def test_one_observation_two_dimensional_draws(ref_loop):
    """A proposal of (n, D) draws, as the restricted prior's: the samples come back (num_samples, D)."""
    res = []
    for loop in (ref_loop, accept_reject_sample):
        prop = Proposal(batch=())
        res.append((*loop(prop, Scripted(0.4), num_samples=700, max_sampling_batch_size=300), prop.sizes))
    (rs, rr, rsz), (s, r, sz) = res
    assert s.shape == (700, 2) and torch.equal(s, rs) and torch.equal(r, rr) and sz == rsz


@needs_ref
@pytest.mark.parametrize("correction, alternative", [(False, None), (False, "sample_with='sir'"), (True, None)])
def test_low_acceptance_warning(ref_loop, caplog, correction, alternative):
    kw = dict(num_samples=40, max_sampling_batch_size=2000, sample_for_correction_factor=correction,
              alternative_method=alternative)
    (rs, rr, rsz, rlog), (s, r, sz, log) = _both(ref_loop, (0.004,), caplog, **kw)
    assert torch.equal(s, rs) and torch.equal(r, rr) and sz == rsz
    # one warning, in the same round: the same rate and the same remaining count
    pat = (r"only\s+([\d.]+%) posterior samples are within.*?remaining\s+(-?\d+) samples" if correction else
           r"Only\s+([\d.]+%) proposal samples are\s+accepted.*?remaining\s+(-?\d+) samples")
    want, got = re.findall(pat, rlog, re.S | re.I), re.findall(pat, log, re.S)
    assert len(want) == 1 and got == want, (rlog, log)
    rate, remaining = want[0]
    if correction:
        assert ("Drawing samples from posterior to estimate the normalizing constant for `log_prob()`. However, "
                f"only {rate} posterior samples are within the prior support. It may take a long time to collect "
                f"the remaining {remaining} samples.") in log
    else:
        msg = (f"Only {rate} proposal samples are accepted. It may take a long time to collect the remaining "
               f"{remaining} samples.")
        if alternative is not None:
            msg += f" Alternatively, consider switching to `{alternative}`."
        assert msg in log and ("consider switching" in log) == (alternative is not None)
    # above the threshold nothing is logged
    caplog.clear()
    with caplog.at_level(logging.WARNING):
        accept_reject_sample(Proposal(), Scripted(0.5), num_samples=40, max_sampling_batch_size=2000)
    assert caplog.text == ""


def test_unused_kwargs_are_logged(caplog):
    with caplog.at_level(logging.WARNING):
        accept_reject_sample(Proposal(), Scripted(1.0), num_samples=5, bogus=3)
    assert "Unused arguments passed to accept_reject_sample: ['bogus']" in caplog.text


def _accepted_rows(prop, fn_thresholds, obs):
    """The accepted draws of observation `obs`, in draw order, under `Scripted(*fn_thresholds)`."""
    rows = []
    for k, d in enumerate(prop.draws):
        p = fn_thresholds[min(k, len(fn_thresholds) - 1)]
        rows.append(d[:, obs][d[:, obs, 0] < (p[obs] if isinstance(p, tuple) else p)])
    return torch.cat(rows)


def test_timeout_with_and_without_a_partial_result():
    # nothing accepted: an error whether or not a partial result is asked for
    for partial in (False, True):
        with pytest.raises(RuntimeError, match="exceeded max_sampling_time"):
            accept_reject_sample(Proposal(delay=0.01), Scripted(0.0), num_samples=10, max_sampling_time=0.02,
                                 return_partial_on_timeout=partial)
    # some accepted: the first rows collected, with the rate so far, and a warning
    prop = Proposal(delay=0.01)
    with pytest.warns(UserWarning, match=r"Timeout exceeded after collecting (\d+)/100000 samples"):
        s, r = accept_reject_sample(prop, Scripted(0.5), num_samples=100_000, max_sampling_batch_size=200,
                                    max_sampling_time=0.05, return_partial_on_timeout=True)
    want = _accepted_rows(prop, (0.5,), 0)
    assert 0 < s.shape[0] == want.shape[0] < 100_000 and s.shape[1:] == (1, 2)
    assert torch.equal(s[:, 0], want)
    assert torch.equal(r, torch.tensor([want.shape[0]]).float() / sum(prop.sizes))
    with pytest.raises(RuntimeError, match="exceeded max_sampling_time"):
        accept_reject_sample(Proposal(delay=0.01), Scripted(0.5), num_samples=100_000, max_sampling_batch_size=200,
                             max_sampling_time=0.05)
    # the clock is checked before every draw but the first
    prop = Proposal(delay=0.001)
    with pytest.raises(RuntimeError, match="exceeded max_sampling_time"):
        accept_reject_sample(prop, Scripted(0.0), num_samples=10, max_sampling_time=0.0)
    assert len(prop.draws) == 1


def test_three_observations():
    """Per observation, the first `num_samples` accepted draws in draw order; the rate per observation; batch sizes
    from what the least-filled observation still needs and the smallest rate."""
    thresholds = ((0.9, 0.3, 0.05), (0.0, 1.0, 0.02), (0.6, 0.1, 0.08))

    class PerObs(Scripted):
        def __call__(self, th):
            p = torch.tensor(self.p[min(self.calls, len(self.p) - 1)])
            self.calls += 1
            return (th[..., 0] < p).reshape(-1)

    num_samples, max_batch = 500, 3000
    prop = Proposal(batch=(3,))
    s, r = accept_reject_sample(prop, PerObs(*thresholds), num_samples=num_samples, num_xos=3,
                                max_sampling_batch_size=max_batch)
    assert s.shape == (num_samples, 3, 2) and r.shape == (3,) and r.dtype == torch.float32
    accepted = [_accepted_rows(prop, thresholds, j) for j in range(3)]
    for j in range(3):
        assert torch.equal(s[:, j], accepted[j][:num_samples]), j
    drawn = sum(prop.sizes)
    assert torch.equal(r, torch.tensor([a.shape[0] for a in accepted]).float() / drawn)
    # replay the batch-size rule on the recorded draws
    want, counts, n = [min(num_samples, max_batch)], torch.zeros(3, dtype=torch.int64), 0
    for k, d in enumerate(prop.draws[:-1]):
        p = torch.tensor(thresholds[min(k, len(thresholds) - 1)])
        counts += (d[..., 0] < p).sum(0)
        n += d.shape[0]
        remaining = num_samples - int(counts.min())
        assert remaining > 0
        rate = float((counts.float() / n).min())
        want.append(min(max_batch, max(int(1.5 * remaining / max(rate, 1e-12)), 100)))
    assert prop.sizes == want and len(want) >= 3


def test_device_argument():
    """With `device`, the accept function sees the candidates there and the counts and rates are kept on the host;
    on the CPU that is the loop without `device`, draw for draw."""
    seen = []

    def accept(th):
        seen.append(th.device)
        return (th[..., 0] < 0.3).reshape(-1)

    runs = []
    for kw in (dict(), dict(device="cpu"), dict(device=torch.device("cpu"))):
        prop = Proposal()
        runs.append((*accept_reject_sample(prop, accept, num_samples=500, max_sampling_batch_size=200, **kw),
                     prop.sizes))
    (s, r, sz) = runs[0]
    for s2, r2, sz2 in runs[1:]:
        assert torch.equal(s2, s) and torch.equal(r2, r) and sz2 == sz
        assert r2.device.type == "cpu" and r2.dtype == torch.float32
    assert len(sz) > 2 and all(d.type == "cpu" for d in seen)
