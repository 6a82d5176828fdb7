"""Wall time of `run_sbc` with batched sampling (`use_batched_sampling=True`: one `sample_batched` call for all
observations) against the per-observation loop (`False`: one `sample` call per observation), on the
linear-Gaussian task (theta 3-d, x = theta A + 0.3 eps 10-d, prior N(0, I)), 200 observations, 1000 draws each.
Posteriors: NLE-`nsf` and NRE-`resnet` (slice MCMC, 20 chains per observation, 50 warm-up steps, thin 2) and FMPE
(ODE and SDE).  The two modes run alternately, in the same process, `--reps` times each; the script prints the
card name and power limit first.  Training time is not part of the measurement.

    python profiles/sbc_time.py [--obs 200] [--draws 1000] [--reps 1]"""
import argparse
import os
import subprocess
import sys
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sbi_b200.diagnostics import run_sbc  # noqa: E402
from sbi_b200.inference import FMPE, NLE, NRE_B  # noqa: E402

MCMC = dict(num_chains=20, warmup_steps=50, thin=2)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def task(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    prior = torch.distributions.MultivariateNormal(torch.zeros(3), torch.eye(3))
    A = torch.randn(3, 10, generator=g) / 3 ** 0.5
    theta = torch.randn(n, 3, generator=g)
    return prior, A, theta, theta @ A + 0.3 * torch.randn(n, 10, generator=g)


def posteriors(prior, theta, x):
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf = NLE(prior, density_estimator="nsf", device="cuda")
        inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=30)
        out["NLE-nsf"] = inf.build_posterior(mcmc_parameters=MCMC)
        inf = NRE_B(prior, classifier="resnet", device="cuda")
        inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=20)
        out["NRE-resnet"] = inf.build_posterior(mcmc_parameters=MCMC)
        inf = FMPE(prior, device="cuda")
        inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=30)
        out["FMPE-ode"] = inf.build_posterior(sample_with="ode")
        out["FMPE-sde"] = inf.build_posterior(sample_with="sde")
    return out


def timed_sbc(post, th, xs, draws, batched):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ranks, _ = run_sbc(th, xs, post, num_posterior_samples=draws, use_batched_sampling=batched)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, ranks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--obs", type=int, default=200)
    ap.add_argument("--draws", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sbc_time.py measures on a GPU; none is visible")
    print("card:", card(), flush=True)
    prior, A, theta, x = task(10_000)
    posts = posteriors(prior, theta, x)
    _, _, th, xs = task(a.obs, seed=1)
    for name, post in posts.items():
        timed_sbc(post, th[:2], xs[:2], 100, True)               # warm-up: kernels loaded, graphs captured once
        times = {True: [], False: []}
        for rep in range(a.reps):
            for batched in ((False, True) if rep % 2 == 0 else (True, False)):
                sec, ranks = timed_sbc(post, th, xs, a.draws, batched)
                times[batched].append(sec)
                print(f"{name:11s} batched={batched!s:5s} {sec:8.2f} s  (mean rank / draws "
                      f"{(ranks.float().mean() / a.draws).item():.3f})", flush=True)
        tb, tl = min(times[True]), min(times[False])
        print(f"{name:11s} {a.obs} obs x {a.draws} draws: batched {tb:.2f} s, loop {tl:.2f} s, "
              f"loop / batched {tl / tb:.2f}", flush=True)


if __name__ == "__main__":
    main()
