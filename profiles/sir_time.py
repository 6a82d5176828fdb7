"""SIR posterior samples per second: `samplers.sampling_importance_resampling` (selection kernel in
csrc/compact.cu) against the reference's loop (sbi/samplers/importance/sir.py, through oracle.ref_shim) driving
the SAME potential, so only the selection differs.  Two potentials: NLE-NSF on the linear-Gaussian task (D = 10)
and the cfg5 NRE-B `resnet` classifier (D = 10).  N = 10^5 samples, K = 32 candidates per sample, batches of
10 000 samples (320 000 potential rows), the two loops alternated in one process after a warm-up.  Then the
selection alone on one 320 000-row batch: our three launches against the reference's softmax / cumsum / mask /
boolean index.  Prints the card name and power limit with the numbers.

    python profiles/sir_time.py [--samples N] [--reps R]
"""
import argparse
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torch.distributions import MultivariateNormal  # noqa: E402

from oracle import ref_shim  # noqa: E402
from sbi_b200 import _lib as L  # noqa: E402
from sbi_b200.neural_nets import likelihood_nn  # noqa: E402
from sbi_b200.posteriors import prior_to_device  # noqa: E402
from sbi_b200.potentials import likelihood_estimator_based_potential, ratio_estimator_based_potential  # noqa: E402
from sbi_b200.ratio import classifier_nn  # noqa: E402
from sbi_b200.samplers import sampling_importance_resampling  # noqa: E402


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
    ap.add_argument("--samples", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sir_time.py measures on a CUDA device")
    assert ref_shim.install(), "needs the reference staged under oracle/_ref by build()"
    from sbi.samplers.importance.sir import sampling_importance_resampling as ref_sir

    D, K, B, N = 10, 32, 10_000, args.samples
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((4000,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    x_o = x[:1]
    proposal = prior_to_device(prior, "cuda")
    pots = {
        "NLE-NSF": likelihood_estimator_based_potential(likelihood_nn("nsf")(theta, x).cuda(), prior, x_o=x_o)[0],
        "NRE-B resnet": ratio_estimator_based_potential(classifier_nn("resnet")(theta, x).cuda(), prior,
                                                        x_o=x_o)[0],
    }
    print(f"card: {card()}")
    print(f"N = {N} samples, K = {K}, batch {B} samples ({B * K} potential rows)")
    for name, op in pots.items():
        pot = lambda t, op=op: op(t, track_gradients=False)   # noqa: E731
        loops = {
            "sbi_b200": lambda n: sampling_importance_resampling(pot, proposal, num_samples=n,
                                                                 num_candidate_samples=K,
                                                                 max_sampling_batch_size=B, device="cuda"),
            "reference": lambda n: ref_sir(pot, proposal, num_samples=n, num_candidate_samples=K,
                                           max_sampling_batch_size=B, device="cuda"),
        }
        for fn in loops.values():                               # warm-up: every batch shape of the timed runs
            fn(2 * B)
        times = {k: [] for k in loops}
        for _ in range(args.reps):
            for k, fn in loops.items():
                t, out = timed(lambda fn=fn: fn(N))
                assert out.shape == (N, D)
                times[k].append(t)
        line = ", ".join(f"{k} {N / min(v):,.0f} samples/s (best of {len(v)}: {min(v) * 1e3:.1f} ms)"
                         for k, v in times.items())
        print(f"{name}: {line}; speed-up {min(times['reference']) / min(times['sbi_b200']):.2f}x")

    # the selection alone on one batch of B groups of K candidates
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(1)
    cand = torch.randn(B * K, D, device="cuda", generator=g)
    lt = torch.randn(B * K, device="cuda", generator=g)
    lq = torch.randn(B * K, device="cuda", generator=g)
    u = torch.rand(B, 1, device="cuda", generator=g)
    out = torch.empty(B, D, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    scratch = torch.empty(int(lib.sbi_b200_sir_scratch_ints(B)), dtype=torch.int32, device="cuda")

    def ours():
        count.zero_()
        L.check(lib.sbi_b200_sir_select(cand.data_ptr(), D, lt.data_ptr(), lq.data_ptr(), u.data_ptr(), B, K, 0,
                                        out.data_ptr(), None, B, count.data_ptr(), scratch.data_ptr(),
                                        L.stream_ptr()), "sir_select")

    def reference():
        w = (lt - lq).reshape(B, K).softmax(-1).cumsum(-1)
        mask = torch.cumsum(w >= u, -1) == 1
        return cand.reshape(B, K, -1)[mask]

    iters = 200
    for fn in (ours, reference):
        fn()
    res = {}
    for name, fn in (("sbi_b200", ours), ("reference", reference)):
        t, _ = timed(lambda fn=fn: [fn() for _ in range(iters)])
        res[name] = t / iters
    nsel = int(count.item())
    # bytes the selection needs: two fp32 log weights per candidate, u per group, and per selected row its D floats
    # read and written (no index output here)
    hbm = (8 * B * K + 4 * B + 8 * D * nsel) / res["sbi_b200"]
    print(f"selection of one batch ({B} groups x {K}, D = {D}): sbi_b200 {res['sbi_b200'] * 1e6:.1f} us "
          f"({hbm / 1e9:.0f} GB/s of weight and row traffic), reference expression "
          f"{res['reference'] * 1e6:.1f} us (with its host sync)")


if __name__ == "__main__":
    main()
