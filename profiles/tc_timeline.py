"""Phase timeline of CTA 0 of the tensor-core training pair (tuning build -DSBI_TC_TIMELINE).
    python profiles/tc_timeline.py [--flush]    # builds sbi_b200/lib/libsbi_b200_tl.so, runs B = 4096, prints deltas
--flush zeroes a 256 MiB buffer before the traced step, as bench.py does before every timed step, so that the
prologue's index and row loads come from HBM; without it the traced step runs with a warm L2.
Prologue markers: forward 1 entry, 2 bias table, 3 ld_const, 4 row gather, 6 first weight stage in; backward
10 entry, 100 first weight stages requested.  They are thread 0's: work another warp still has in hand shows up at
the next CTA barrier."""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sbi_b200 import build as _b
lib_path = os.path.join(ROOT, "sbi_b200", "lib", "libsbi_b200_tl.so")
if "--build" in sys.argv or not os.path.exists(lib_path):
    _b.build_variant("tl", ["SBI_TC_TIMELINE"])
if "--build-only" in sys.argv:
    sys.exit(0)
os.environ["SBI_B200_LIB"] = lib_path
import torch
from bench import DIM, NUM_SIMS, make_data
from sbi_b200 import _lib as L
from sbi_b200.neural_nets import posterior_nn
B = 4096
lib = L.load()
theta, x = make_data(NUM_SIMS, DIM)
torch.manual_seed(0)
est = posterior_nn("nsf")(theta[:90000], x[:90000]).cuda()
th, xx = theta.cuda(), x.cuda()
idx = torch.randperm(90000, device="cuda")[:B]
m = est._model(nbuf=3)
rows = L.Rows(th.data_ptr(), xx.data_ptr(), idx.data_ptr(), B, 0)
lp = torch.empty(B, device="cuda")
acc = torch.zeros(2, device="cuda")
os.environ["SBI_B200_VJP_TC"] = "1"
gpart = est._gpart(est.vjp_parts(B))
run = lambda: est.vjp(m, rows, B, None, -1.0 / B, lp, gpart, None, None, acc)
buf = (C.c_ulonglong * 8192)()
for name in ("fwd", "bwd"):
    getattr(lib, f"sbi_b200_debug_timeline_{name}").restype = C.c_int
for _ in range(3):
    run()
torch.cuda.synchronize()
for name in ("fwd", "bwd"):
    getattr(lib, f"sbi_b200_debug_timeline_{name}")(buf, 4096)          # reset
if "--flush" in sys.argv:
    torch.empty(256 << 20, dtype=torch.uint8, device="cuda").zero_()
run()
torch.cuda.synchronize()
for name in ("fwd", "bwd"):
    n = getattr(lib, f"sbi_b200_debug_timeline_{name}")(buf, 4096)
    ev = [(int(buf[2 * i]), int(buf[2 * i + 1])) for i in range(n)]
    print(f"## {name}: {n} marks, total {(ev[-1][1] - ev[0][1]) / 1965:.1f} us (clock64 / 1965 MHz)")
    prev = ev[0][1]
    line = []
    for i, t in ev:
        line.append(f"{i}:{(t - prev) / 1965:.2f}")
        prev = t
        if len(line) == 12:
            print("  " + "  ".join(line)); line = []
    if line:
        print("  " + "  ".join(line))
