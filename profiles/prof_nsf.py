"""Launch the NSF kernels a few times on the bench workload (for ncu captures)."""
import ctypes as C
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import BATCH, DIM, NUM_SIMS, make_data  # noqa: E402
from sbi_b200 import _lib as L  # noqa: E402
from sbi_b200.neural_nets import posterior_nn  # noqa: E402

which = sys.argv[1] if len(sys.argv) > 1 else "all"
lib = L.load()
theta, x = make_data(NUM_SIMS, DIM)
torch.manual_seed(0)
est = posterior_nn("nsf")(theta[:90000], x[:90000]).cuda()
th, xx = theta.cuda(), x.cuda()
P = est.layout.n_params
n_part = lib.sbi_b200_nsf_vjp_parts(BATCH)
gpart = est._gpart(n_part)
grad = torch.zeros(P, device="cuda"); state = torch.zeros(2 * P, device="cuda")
step = torch.zeros(2, dtype=torch.int32, device="cuda")
idx = torch.randperm(90000, device="cuda")[:BATCH]
save = torch.empty(lib.sbi_b200_nsf_vjp_save_bytes(C.byref(est._model(nbuf=3)), BATCH) // 4, device="cuda")
for it in range(4):
    if which in ("all", "vjp"):
        m = est._model(nbuf=3)
        rows = L.Rows(th.data_ptr(), xx.data_ptr(), idx.data_ptr(), BATCH, 0)
        L.check(lib.sbi_b200_nsf_vjp(C.byref(m), C.byref(rows), None, -1.0 / BATCH, None, L.ptr(gpart), None, None,
                                     None, L.ptr(save), save.numel() * 4, L.stream_ptr()), "vjp")
        L.check(lib.sbi_b200_reduce_partials(L.ptr(gpart), n_part, P, L.ptr(grad), L.stream_ptr()), "red")
        L.check(lib.sbi_b200_adam_clip_step(L.ptr(est.flat.data), L.ptr(grad), L.ptr(state), L.ptr(step),
                                            L.ptr(est.net._mask), P, 5e-4, .9, .999, 1e-8, 5.0, 1.0, L.stream_ptr()), "adam")
    if which in ("all", "logprob"):
        R = 1 << 21
        te = math.sqrt(0.1) * torch.randn(R, DIM, device="cuda")
        est._logprob_raw(te, xx[:1].contiguous(), True)
    if which in ("all", "inverse"):
        est.sample((1 << 20,), xx[:1])
torch.cuda.synchronize()
print("done")
