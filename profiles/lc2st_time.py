"""L-C2ST wall times: `sbi_b200.diagnostics.LC2ST` (training and evaluation kernels in csrc/lc2st.cu) against the
reference's scikit-learn path (sbi/diagnostics/lc2st.py through oracle.ref_shim) on the same inputs, the two
alternated in one process.  Per configuration (dim_theta 2 / N 1 000 and dim_theta 5 / N 10 000, dim_x =
dim_theta, default classifier, 100 null trials): `train_on_observed_data` + `train_under_null_hypothesis`, then
100 `reject_test` calls at one observation with 1 000 theta_o rows; then the kernel times of one training launch and
one evaluation launch from torch.profiler.  The reference at N 10 000 takes minutes on the CPU, so it only runs
there with --ref-big.  Prints the card name and power limit, and the CPU model and the cores the reference's
sklearn could use, with the numbers: both sides run in the same process on the same host.

    python profiles/lc2st_time.py [--ref-big] [--reps R]
"""
import argparse
import os
import subprocess
import sys
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shim  # noqa: E402
from sbi_b200.diagnostics import LC2ST  # noqa: E402


def _data(d, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(n, d, generator=g)
    x = theta + 0.7 * torch.randn(n, d, generator=g)
    post = x / 1.5 + 0.2 + 0.58 * torch.randn(n, d, generator=g)
    x_o = torch.zeros(d)
    theta_o = x_o / 1.5 + 0.2 + 0.58 * torch.randn(1000, d, generator=g)
    return theta, x, post, theta_o, x_o


def _run(cls, d, n, reject_calls):
    theta, x, post, theta_o, x_o = _data(d, n)
    lc = cls(theta, x, post)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lc.train_on_observed_data(seed=1, verbosity=0).train_under_null_hypothesis(verbosity=0)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        for _ in range(reject_calls):
            lc.reject_test(theta_o=theta_o, x_o=x_o)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
    return t1 - t0, t2 - t1, lc


def _kernel_times(d, n):
    from torch.profiler import ProfilerActivity, profile
    theta, x, post, theta_o, x_o = _data(d, n)
    lc = LC2ST(theta, x, post)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        lc.train_on_observed_data(seed=1)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            lc.train_under_null_hypothesis()
            torch.cuda.synchronize()
            lc.reject_test(theta_o=theta_o, x_o=x_o)
            torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "lc2st" in e.key:
            out[e.key.split("(")[0].split("::")[-1]] = e.device_time_total / 1e3 / max(e.count, 1)
    return out, [c.n_iter_ for t in range(lc.num_trials_null) for c in lc.trained_clfs_null[t]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref-big", action="store_true", help="also run the reference at dim_theta 5 / N 10 000")
    ap.add_argument("--reps", type=int, default=1)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    cpu = next((ln.split(":", 1)[1].strip() for ln in open("/proc/cpuinfo") if ln.startswith("model name")), "?")
    cores = len(os.sched_getaffinity(0))
    print(f"device: {card}; host CPU: {cpu}, {cores} cores available to this process, torch threads "
          f"{torch.get_num_threads()}")
    ref = None
    if ref_shim.available() and ref_shim.install():
        from sbi.diagnostics.lc2st import LC2ST as ref
    _run(LC2ST, 2, 200, 1)   # warm-up: library load, kernel attributes
    for d, n in ((2, 1000), (5, 10000)):
        for rep in range(args.reps):
            tr, ev, lc = _run(LC2ST, d, n, 100)
            it = [c.n_iter_ for t in range(lc.num_trials_null) for c in lc.trained_clfs_null[t]]
            print(f"ours  d={d} N={n}: train (observed + 100 null) {tr:8.2f} s, 100 reject_test {ev:7.2f} s; "
                  f"null epochs min/median/max {min(it)}/{sorted(it)[len(it) // 2]}/{max(it)}")
            if ref is not None and (n <= 1000 or args.ref_big):
                tr_r, ev_r, lc_r = _run(ref, d, n, 100)
                it = [c.n_iter_ for t in range(lc_r.num_trials_null) for c in lc_r.trained_clfs_null[t]]
                print(f"ref   d={d} N={n}: train (observed + 100 null) {tr_r:8.2f} s, 100 reject_test {ev_r:7.2f} s; "
                      f"null epochs min/median/max {min(it)}/{sorted(it)[len(it) // 2]}/{max(it)}")
        k, it = _kernel_times(d, n)
        print(f"kernels d={d} N={n} (ms per launch): " + ", ".join(f"{a} {b:.2f}" for a, b in sorted(k.items())) +
              f"; the training launch runs until the slowest of its 100 models stops ({max(it)} epochs)")


if __name__ == "__main__":
    main()
