"""Time the NSF kernels of the bench workload for the library selected by $SBI_B200_LIB."""
import ctypes as C
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import BATCH, DIM, NUM_SIMS, make_data  # noqa: E402
from sbi_b200 import _lib as L  # noqa: E402
from sbi_b200.neural_nets import posterior_nn  # noqa: E402

lib = L.load()
theta, x = make_data(NUM_SIMS, DIM)
torch.manual_seed(0)
est = posterior_nn("nsf")(theta[:90000], x[:90000]).cuda()
th, xx = theta.cuda(), x.cuda()
P = est.layout.n_params
n_part = lib.sbi_b200_nsf_vjp_parts(BATCH)
gpart = est._gpart(n_part)
idx = torch.randperm(90000, device="cuda")[:BATCH]
save = torch.empty(lib.sbi_b200_nsf_vjp_save_bytes(C.byref(est._model(nbuf=3)), BATCH) // 4, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
nbuf_tr = int(os.environ.get("NBUF_TRAIN", "3"))
nbuf_ev = int(os.environ.get("NBUF_EVAL", "2"))


def timeit(fn, n=20, do_flush=True):
    for _ in range(3):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for a, b in ev:
        if do_flush:
            flush.zero_()
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in ev)
    return t[len(t) // 2]


def vjp():
    m = est._model(nbuf=nbuf_tr)
    rows = L.Rows(th.data_ptr(), xx.data_ptr(), idx.data_ptr(), BATCH, 0)
    L.check(lib.sbi_b200_nsf_vjp(C.byref(m), C.byref(rows), None, -1.0 / BATCH, None, L.ptr(gpart), None, None, None,
                                 L.ptr(save), save.numel() * 4, L.stream_ptr()), "vjp")


R = 1 << 22
te = math.sqrt(0.1) * torch.randn(R, DIM, device="cuda")
xo = xx[:1].contiguous()
lp = torch.empty(R, device="cuda")


def logprob():
    m = est._model(nbuf=nbuf_ev)
    rows = L.Rows(te.data_ptr(), xo.data_ptr(), None, R, 1)
    L.check(lib.sbi_b200_nsf_logprob(C.byref(m), C.byref(rows), L.ptr(lp), None, L.stream_ptr()), "lp")


print(f"{os.environ.get('SBI_B200_LIB', 'default')} nbuf={nbuf_tr}/{nbuf_ev}: "
      f"vjp {timeit(vjp) * 1e3:.1f} us   logprob(4.2M rows) {timeit(logprob, n=8, do_flush=False):.2f} ms")
