"""First-light check of the tensor-core training kernels (run under `timeout`): one 128-row tile, then
4096 rows, gradients vs the SIMT kernel; prints per-tensor errors."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.helpers import b200_from_oracle, oracle_nsf, use_vjp_path, vjp_step  # noqa: E402

D, C = 10, 10
flow, theta, x = oracle_nsf(D, C, n=5000)
est = b200_from_oracle(flow, theta, x)
for R in (128, 300, 4096):
    inp, cond = (theta[:R] * 1.3).float().cuda().contiguous(), x[:R].float().cuda().contiguous()
    g = torch.randn(R).cuda()
    with pytest.MonkeyPatch.context() as mp:
        use_vjp_path(mp, est, False)
        s = vjp_step(est, inp, cond, g, tc=False)
        print("simt done", flush=True)
        use_vjp_path(mp, est, True)
        t = vjp_step(est, inp, cond, g)
    simt, tc = s.grad.double(), t.grad.double()
    print(f"R={R} n_part={t.gpart.shape[0]} logp diff {(t.logp - s.logp).abs().max():.3e} "
          f"acc {t.loss_acc.tolist()} vs {s.loss_acc.tolist()}", flush=True)
    sc = simt.abs().max()
    print(f"   grad: max|simt| {sc:.3e}  max diff {(tc - simt).abs().max():.3e}  nan {int(torch.isnan(tc).sum())}")
    for name, idx in est.layout.index.items():
        i = torch.as_tensor(idx.reshape(-1))
        d = (tc[i] - simt[i]).abs().max().item()
        s_ = simt[i].abs().max().item()
        if d > 2e-3 * sc or not (d == d):
            print(f"   {name:70s} diff {d:.3e} (|ref| {s_:.3e})")
print("done")
