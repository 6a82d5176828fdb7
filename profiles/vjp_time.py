"""Kernel time of nsf_vjp (activation spill to a caller-owned scratch) at the bench shape (B = 4096, dim 10): CUDA
events around the launch."""
import ctypes as C, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import BATCH, DIM, NUM_SIMS, make_data
from sbi_b200 import _lib as L
from sbi_b200.neural_nets import posterior_nn
lib = L.load()
theta, x = make_data(NUM_SIMS, DIM)
torch.manual_seed(0)
est = posterior_nn("nsf")(theta[:90000], x[:90000]).cuda()
th, xx = theta.cuda(), x.cuda()
n_part = lib.sbi_b200_nsf_vjp_parts(BATCH)
gpart = est._gpart(n_part)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
idx = torch.randperm(90000, device="cuda")[:BATCH]
m = est._model(nbuf=3)
rows = L.Rows(th.data_ptr(), xx.data_ptr(), idx.data_ptr(), BATCH, 0)
save = torch.empty(lib.sbi_b200_nsf_vjp_save_bytes(C.byref(m), BATCH) // 4, device="cuda")
def run():
    L.check(lib.sbi_b200_nsf_vjp(C.byref(m), C.byref(rows), None, -1.0 / BATCH, None, L.ptr(gpart), None, None,
                                 None, L.ptr(save), save.numel() * 4, L.stream_ptr()), "vjp")
for _ in range(5): run()
torch.cuda.synchronize()
ts = []
for _ in range(30):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); run(); e1.record(); torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
ts.sort()
print(f"nsf_vjp B={BATCH}: median {ts[len(ts)//2]*1e3:.1f} us  min {ts[0]*1e3:.1f} us")
