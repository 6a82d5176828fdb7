"""NUTS / HMC lock-step times and effective samples per second against the slice sampler.

For NLE-`nsf` and NRE-B `resnet` potentials on the linear-Gaussian task (D = 2 and 10, briefly trained: only the
cost matters here) and 20 or 1 000 chains, prints:
  * the lock-step time of a NUTS run under graph replay (wall time of `run` over its lock-steps),
  * the potential+gradient part alone (a CUDA graph of 16 evaluations, CUDA events), the state-machine kernel as
    the difference, and the forward-only potential (the share a fused value+gradient launch could save: today the
    VJP kernel recomputes the forward),
  * effective samples per second of `nuts_pyro` and `slice_np_vectorized` (their defaults: thin 1 and 10, 200
    warm-up transitions / sweeps) on the same potential, with the ESS from batch means pooled over chains (the
    minimum over dimensions).
Prints the card name and its power limit.

    python profiles/hmc_time.py [--samples N]
"""
import argparse
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sbi_b200.hmc import HMCSamplerVectorized, frozen_parameters  # noqa: E402
from sbi_b200.inference import NLE, NRE_B  # noqa: E402
from sbi_b200.potentials import transformed_potential  # noqa: E402


def batch_means_ess(s: np.ndarray) -> float:
    """(chains, n, D) -> min over dimensions of N var / (b var(batch means)), batches of b = floor(sqrt(n))."""
    C, n, D = s.shape
    b = max(1, int(math.sqrt(n)))
    k = n // b
    bm = s[:, :k * b].reshape(C, k, b, D).mean(2).reshape(-1, D)
    var = s[:, :k * b].reshape(-1, D).var(0, ddof=1)
    return float(np.min(C * k * b * var / (b * bm.var(0, ddof=1))))


def _trained(kind, D):
    torch.manual_seed(0)
    prior = torch.distributions.MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((5000,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    tr = NLE(prior, density_estimator="nsf", device="cuda") if kind == "nle" else \
        NRE_B(prior, classifier="resnet", device="cuda")
    tr.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=10)
    return tr, x[:1]


def _graph_time(fn, reps=16, iters=20):
    fn()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        for _ in range(reps):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (iters * reps)     # microseconds per evaluation


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=2000)
    args = ap.parse_args()
    name = torch.cuda.get_device_name()
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip().splitlines()
    print(f"# {name}, power limit {power[0] if power else 'unknown'}")
    print("kind D chains | lockstep_us pot+grad_us kernel_us fwd_only_us | nuts_ess/s slice_ess/s "
          "(nuts ess, s | slice ess, s) depth")
    for kind in ("nle", "nre"):
        for D in (2, 10):
            tr, x_o = _trained(kind, D)
            for C in (20, 1000):
                post = tr.build_posterior(mcmc_method="nuts_pyro", mcmc_parameters=dict(num_chains=C))
                post.potential_fn.set_x(x_o, x_is_iid=True)
                pot, tf = post.potential_fn, post.theta_transform
                params = tf(post.proposal.sample((C,))).float().contiguous()

                def lp_fn(p):
                    return transformed_potential(p, pot, tf, "cuda", track_gradients=True).flatten()

                def pot_grad():
                    with torch.enable_grad():
                        p = params.detach().requires_grad_(True)
                        torch.autograd.grad(lp_fn(p).sum(), p)

                def fwd_only():
                    with torch.no_grad():
                        transformed_potential(params, pot, tf, "cuda", track_gradients=False)

                with frozen_parameters(pot):
                    t_pg = _graph_time(pot_grad)
                    t_f = _graph_time(fwd_only)
                    smp = HMCSamplerVectorized(lp_fn, params.double(), num_chains=C, warmup_steps=200, graph=True)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    smp.run(100)
                    torch.cuda.synchronize()
                    t_ls = (time.perf_counter() - t0) * 1e6 / smp.num_lock_steps
                n = args.samples if C == 20 else 20 * args.samples
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                post.sample((n,), x=x_o)
                torch.cuda.synchronize()
                t_nuts = time.perf_counter() - t0
                ess_nuts = batch_means_ess(post._posterior_sampler.get_samples())
                depth = float(np.mean(post._posterior_sampler.mean_tree_depth))
                sl = tr.build_posterior(mcmc_method="slice_np_vectorized", mcmc_parameters=dict(num_chains=C))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                sl.sample((n,), x=x_o)
                torch.cuda.synchronize()
                t_slice = time.perf_counter() - t0
                raw = sl._posterior_sampler.get_samples()[:, 200:, :]     # thinned sweeps after warm-up
                ess_slice = batch_means_ess(raw)
                print(f"{kind} {D:2d} {C:5d} | {t_ls:9.1f} {t_pg:9.1f} {t_ls - t_pg:9.1f} {t_f:9.1f} | "
                      f"{ess_nuts / t_nuts:10.0f} {ess_slice / t_slice:10.0f} "
                      f"({ess_nuts:.0f}, {t_nuts:.2f} | {ess_slice:.0f}, {t_slice:.2f}) {depth:.2f}", flush=True)


if __name__ == "__main__":
    main()
