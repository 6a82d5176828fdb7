"""Kernel times of the tensor-core training step, one line per kernel: operand pack (tc_pack_kernel),
forward sweep with activation save (nsf_logprob_tc_kernel<..., SAVE>), backward sweep (nsf_vjp_tc_kernel) and
weight-gradient kernel (nsf_dw_tc_kernel), at the bench model (cfg2: NSF dim 10) and 4096 / 32768 rows, L2
flushed before every step.  Kernel times come from torch.profiler (CUDA activities), the step time from CUDA
events in a separate, unprofiled loop.
    python profiles/vjp_tc_split_time.py [steps]"""
import os, sys
from collections import defaultdict
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import DIM, NUM_SIMS, make_data
from sbi_b200 import _lib as L
from sbi_b200.neural_nets import posterior_nn

STEPS = int(sys.argv[1]) if len(sys.argv) > 1 else 50
KERNELS = (("pack", "tc_pack_kernel"), ("forward", "nsf_logprob_tc_kernel"), ("backward", "nsf_vjp_tc_kernel"),
           ("dW", "nsf_dw_tc_kernel"))
os.environ["SBI_B200_VJP_TC"] = "1"
theta, x = make_data(NUM_SIMS, DIM)
torch.manual_seed(0)
est = posterior_nn("nsf")(theta[:90000], x[:90000]).cuda()
th, xx = theta.cuda(), x.cuda()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
print(torch.cuda.get_device_name(), flush=True)
for B in (4096, 32768):
    idx = torch.randperm(90000, device="cuda")[:B]
    m = est._model(nbuf=3)
    rows = L.Rows(th.data_ptr(), xx.data_ptr(), idx.data_ptr(), B, 0)
    lp = torch.empty(B, device="cuda")
    acc = torch.zeros(2, device="cuda")
    gpart = est._gpart(est.vjp_parts(B))
    run = lambda: est.vjp(m, rows, B, None, -1.0 / B, lp, gpart, None, None, acc)
    for _ in range(5):
        run()
    torch.cuda.synchronize()
    ts = []
    for _ in range(STEPS):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); run(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(STEPS):
            flush.zero_()
            run()
        torch.cuda.synchronize()
    tot, cnt = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for label, key in KERNELS:
            if key in e.name:
                tot[label] += e.device_time
                cnt[label] += 1
    parts = "  ".join(f"{label} {tot[label] / STEPS:.1f} us ({cnt[label] // STEPS}/step)"
                      for label, _ in KERNELS if cnt[label])
    print(f"B={B}: step median {ts[len(ts) // 2]:.1f} us (min {ts[0]:.1f})  |  {parts}", flush=True)
