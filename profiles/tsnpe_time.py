"""TSNPE's two device-heavy calls at the bench shape (D = C = 10, NSF `DirectPosterior`):

* `get_density_thresholder(posterior)`: 10^6 posterior draws and their log-probs, one sort;
* `RestrictedPrior(prior, thresholder).sample((10 000,))` at an x_o where the prior's acceptance is about 1 % and
  about 0.1 %, against the same accept function called the way `DirectPosterior.sample` calls
  `posteriors.accept_reject_sample` (draws moved to the device inside the proposal, so the acceptance counts stay
  there too), from the same seed and the same prior draws.  Both go through the one loop.

The posterior is NPE trained briefly on the linear-Gaussian task (x = theta + sqrt(0.1) eps, prior N(0, I)); the
x_o's are picked by scanning x_o = s * (1, ..., 1) / sqrt(10) for the estimated acceptance.  Times are CUDA events
around each call with a final synchronise, after a warm-up of every call; the card's name and power limit are
printed with them.

    python profiles/tsnpe_time.py [--reps R]
"""
import argparse
import math
import os
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torch.distributions import MultivariateNormal  # noqa: E402

from sbi_b200.inference import NPE  # noqa: E402
from sbi_b200.posteriors import accept_reject_sample  # noqa: E402
from sbi_b200.restriction import RestrictedPrior, get_density_thresholder  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:   # noqa: BLE001
        pl = "unknown"
    return f"{name}, power limit {pl or 'unknown'}"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tsnpe_time.py measures on a CUDA device")
    D, N, n = 10, 1_000_000, 10_000
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), torch.eye(D))
    theta = prior.sample((20_000,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf = NPE(prior, density_estimator="nsf", device="cuda")
        inf.append_simulations(theta, x).train(max_num_epochs=30)
    print(f"card: {card()}")

    # x_o's whose 1 - 1e-4 posterior region holds about 1 % and 0.1 % of the prior
    probe = prior.sample((200_000,)).cuda()
    found = {}
    for s in [0.25 * i for i in range(25)]:
        x_o = torch.full((1, D), s / math.sqrt(D))
        post = inf.build_posterior().set_default_x(x_o)
        rate = get_density_thresholder(post, num_samples_to_estimate_support=100_000)(probe).float().mean().item()
        for target in (1e-2, 1e-3):
            if rate > 0 and (target not in found or
                             abs(math.log(rate / target)) < abs(math.log(found[target][1] / target))):
                found[target] = (s, rate)
    print("x_o scan (s, estimated acceptance): " + ", ".join(f"{t:g}: {v}" for t, v in found.items()))

    for target, (s, _) in found.items():
        x_o = torch.full((1, D), s / math.sqrt(D))
        post = inf.build_posterior().set_default_x(x_o)
        timed(lambda: get_density_thresholder(post, num_samples_to_estimate_support=N))       # warm-up
        t_thr = []
        for _ in range(args.reps):
            t, thr = timed(lambda: get_density_thresholder(post, num_samples_to_estimate_support=N))
            t_thr.append(t)
        rp = RestrictedPrior(prior, thr, device="cuda")
        loops = {
            "RestrictedPrior.sample": lambda: rp.sample((n,), save_acceptance_rate=True, print_rejected_frac=False),
            "accept_reject_sample, proposal on the device": lambda: accept_reject_sample(
                lambda shape, **kw: prior.sample(shape).cuda(), thr, num_samples=n)[0].reshape(n, D),
        }
        outs, times = {}, {k: [] for k in loops}
        for k, f in loops.items():     # warm-up
            torch.manual_seed(1)
            outs[k] = f()
        same = torch.equal(*[o.cpu() for o in outs.values()])
        for _ in range(args.reps):
            for k, f in loops.items():
                torch.manual_seed(1)
                times[k].append(timed(f)[0])
        print(f"\nx_o = {s:g} * 1/sqrt(10): acceptance {rp.acceptance_rate.item():.4%} "
              f"({n / rp.acceptance_rate.item():.3g} prior draws per call)")
        print(f"  get_density_thresholder (N = {N}): " + ", ".join(f"{t * 1e3:.1f}" for t in t_thr) + " ms")
        for k, ts in times.items():
            print(f"  {k}: " + ", ".join(f"{t * 1e3:.1f}" for t in ts) + " ms")
        print(f"  samples bit-equal between the two calls: {same}")


if __name__ == "__main__":
    main()
