"""Overlap of the weight-gradient kernel (nsf_dw_tc_kernel) with the backward sweep (nsf_vjp_tc_kernel) in the
tensor-core training step, as the trainer runs it: one step captured in a CUDA graph and replayed, at the bench
model (cfg2: NSF dim 10) and 4096 / 32768 rows.  One torch.profiler trace (CUDA activities) of the replays;
per chunk of the step it reports when the dW kernel starts relative to the backward's start and end, and how
long dW runs on after the backward has ended, and when the backward starts relative to the forward's end.  A dW start at or after the backward's end means that the
programmatic launch edge was lost (results stay correct, the overlap is gone).  The trace goes to OUT_DIR.
    python profiles/vjp_tc_overlap.py [OUT_DIR] [replays]"""
import json
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import DIM, NUM_SIMS, make_data  # noqa: E402
from sbi_b200 import _lib as L  # noqa: E402
from sbi_b200.neural_nets import posterior_nn  # noqa: E402

OUT = sys.argv[1] if len(sys.argv) > 1 else tempfile.mkdtemp()
REPLAYS = int(sys.argv[2]) if len(sys.argv) > 2 else 20
os.makedirs(OUT, exist_ok=True)
os.environ["SBI_B200_VJP_TC"] = "1"
theta, x = make_data(NUM_SIMS, DIM)
torch.manual_seed(0)
est = posterior_nn("nsf")(theta[:90000], x[:90000]).cuda()
th, xx = theta.cuda(), x.cuda()
print(torch.cuda.get_device_name(), flush=True)


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


for B in (4096, 32768):
    idx = torch.randperm(90000, device="cuda")[:B]
    m = est._model(nbuf=3)
    rows = L.Rows(th.data_ptr(), xx.data_ptr(), idx.data_ptr(), B, 0)
    lp = torch.empty(B, device="cuda")
    acc = torch.zeros(2, device="cuda")
    gpart = est._gpart(est.vjp_parts(B))
    run = lambda: est.vjp(m, rows, B, None, -1.0 / B, lp, gpart, None, None, acc)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            run()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    for _ in range(5):
        graph.replay()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(REPLAYS):
            graph.replay()
        torch.cuda.synchronize()
    path = os.path.join(OUT, f"vjp_tc_overlap_{B}.json")
    prof.export_chrome_trace(path)
    with open(path) as fh:
        ev = [e for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    # pair every backward with the forward before it and the dW kernel after it (one triple per chunk of the step)
    fwd, bwd, pairs, fb = None, None, [], []
    for e in ev:
        if "nsf_logprob_tc_kernel" in e["name"]:
            fwd = e
        elif "nsf_vjp_tc_kernel" in e["name"]:
            bwd = e
            if fwd is not None:
                fb.append((fwd, e))
                fwd = None
        elif "nsf_dw_tc_kernel" in e["name"] and bwd is not None:
            pairs.append((bwd, e))
            bwd = None
    chunks = len(pairs) // REPLAYS
    for c in range(chunks):
        ps = pairs[c::chunks]
        b_dur = [b["dur"] for b, _ in ps]
        start_rel = [d["ts"] - b["ts"] for b, d in ps]
        start_vs_end = [d["ts"] - (b["ts"] + b["dur"]) for b, d in ps]
        tail = [d["ts"] + d["dur"] - (b["ts"] + b["dur"]) for b, d in ps]
        d_dur = [d["dur"] for _, d in ps]
        print(f"B={B} chunk {c}: backward {median(b_dur):.1f} us | dW starts {median(start_rel):.1f} us after the "
              f"backward's start, {median(start_vs_end):+.1f} us from its end | dW runs {median(d_dur):.1f} us, "
              f"{median(tail):.1f} us past the backward's end (medians of {len(ps)} replays)", flush=True)
    # the backward is launched early behind the forward: its grid starts (first CTA resident) before the forward
    # ends when SMs are free for it (half tiles)
    for c in range(len(fb) // REPLAYS):
        ps = fb[c::len(fb) // REPLAYS]
        f_dur = [f["dur"] for f, _ in ps]
        b_vs_end = [b["ts"] - (f["ts"] + f["dur"]) for f, b in ps]
        print(f"B={B} chunk {c}: forward {median(f_dur):.1f} us | backward starts {median(b_vs_end):+.1f} us from "
              f"the forward's end (medians of {len(ps)} replays)", flush=True)
    print("trace:", path, flush=True)
