"""MMD misspecification test wall times: `sbi_b200.diagnostics.calc_misspecification_mmd` (csrc/mmd.cu) against the
reference's CPU loop (sbi/diagnostics/misspecification.py through oracle.ref_shim) on the same inputs and seed, the
two alternated in one process.  N = 10 000 simulations, n_shuffle = 1 000, max_samples in {1 000, 4 000}, n_obs in
{1, 100}, d in {2, 20, 100}.  Per configuration: the end-to-end call (median of --reps), the host's `randperm`
table alone, and the device launches alone on a prebuilt table (CUDA events).  The reference runs --ref-shuffles
null draws (default 100) at max_samples 1 000 and is reported per 100 shuffles; its cost grows with max_samples^2,
so max_samples 4 000 only runs with --ref-big.  Prints the card name and power limit, and the CPU cores available.

    python profiles/misspec_time.py [--reps R] [--ref-shuffles K] [--ref-big]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shim  # noqa: E402
from sbi_b200 import misspecification as M  # noqa: E402

N, N_SHUFFLE = 10_000, 1_000


def _data(n_obs, d, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n_obs, d, generator=g) + 0.2, torch.randn(N, d, generator=g)


def _device_times(x_o, x, max_samples, reps):
    xo_d, x_d = x_o.cuda(), x.cuda()
    ends = []
    for r in range(reps + 1):
        torch.manual_seed(r)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        M.calc_misspecification_mmd(xo_d, x_d, n_shuffle=N_SHUFFLE, max_samples=max_samples)
        torch.cuda.synchronize()
        if r:
            ends.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    M.shuffle_table(N, N_SHUFFLE, max_samples)
    t_perm = time.perf_counter() - t0
    n_obs, m = x_o.shape[0], min(N, max_samples)
    perms = M.shuffle_table(N, N_SHUFFLE, max_samples).to(torch.int32)
    obs = torch.cat([torch.arange(N, N + n_obs), torch.arange(m)]).to(torch.int32)
    table = torch.cat([torch.nn.functional.pad(perms, (0, n_obs)), obs.unsqueeze(0)])
    nxy = torch.cat([torch.tensor([[n_obs, m - n_obs]]).expand(N_SHUFFLE, 2), torch.tensor([[n_obs, m]])])
    z = torch.cat([x_d, xo_d]).contiguous()
    d_table = table.cuda()
    M._mmd_sets(z, d_table, nxy)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    dev = []
    for _ in range(reps):
        ev[0].record()
        M._mmd_sets(z, d_table, nxy)
        ev[1].record()
        torch.cuda.synchronize()
        dev.append(ev[0].elapsed_time(ev[1]) / 1e3)
    return statistics.median(ends), t_perm, statistics.median(dev)


def _reference_time(R, x_o, x, max_samples, k):
    torch.manual_seed(0)
    t0 = time.perf_counter()
    R.calculate_p_misspecification(x_o, x, n_shuffle=k, max_samples=max_samples)
    return (time.perf_counter() - t0) * 100 / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-shuffles", type=int, default=100)
    ap.add_argument("--ref-big", action="store_true")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"GPU: {card[0] if card else torch.cuda.get_device_name()}; CPU cores available: "
          f"{len(os.sched_getaffinity(0))}, torch threads {torch.get_num_threads()}")
    R = None
    if ref_shim.available():
        ref_shim.install()
        from sbi.diagnostics import misspecification as R
    print("max_samples n_obs   d | device end-to-end   of which randperm   launches | reference per 100 shuffles")
    for max_samples in (1_000, 4_000):
        for n_obs in (1, 100):
            for d in (2, 20, 100):
                x_o, x = _data(n_obs, d)
                t_ref = None
                if R is not None and (max_samples == 1_000 or a.ref_big):
                    t_ref = _reference_time(R, x_o, x, max_samples, a.ref_shuffles)
                end, perm, dev = _device_times(x_o, x, max_samples, a.reps)
                ref = f"{t_ref:8.3f} s" if t_ref is not None else "not run"
                print(f"{max_samples:11d} {n_obs:5d} {d:3d} | {end * 1e3:11.1f} ms {perm * 1e3:15.1f} ms "
                      f"{dev * 1e3:8.2f} ms | {ref}", flush=True)


if __name__ == "__main__":
    main()
