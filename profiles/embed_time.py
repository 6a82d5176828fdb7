"""Cost of training a torch embedding net inside the fused trainers (prints the card name and power limit).

* NPE-`nsf` epoch time, identity embedding vs an FC embedding (x 100-d -> 10), at batch 200 and 4096;
* the 4096-row training VJP three ways: wgmma parameter-only, wgmma with the condition gradient d_gcond (the
  trainer's step with an embedding net from VJP_TC_MIN_ROWS rows on), SIMT with d_gcond (below that, or for
  models the wgmma kernel declines).  Each call re-packs the wgmma operands, as the trainer's step does;
* FMPE epoch time with and without the FC embedding.
Epoch times are the median of the epochs after the first (which includes the graph capture)."""
import ctypes as C
import os
import statistics
import subprocess
import sys

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sbi_b200 import _lib as L  # noqa: E402
from sbi_b200.flowmatching import posterior_flow_nn  # noqa: E402
from sbi_b200.inference import FMPE, NPE  # noqa: E402
from sbi_b200.neural_nets import posterior_nn  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def fc():
    return nn.Sequential(nn.Linear(100, 100), nn.ReLU(), nn.Linear(100, 10))


def data(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(n, 5, generator=g)
    A = torch.randn(5, 100, generator=g) / 5 ** 0.5
    return theta, theta @ A + 0.3 * torch.randn(n, 100, generator=g)


def epoch_ms(trainer, build, n, batch, epochs=6):
    theta, x = data(n)
    torch.manual_seed(0)
    inf = trainer(density_estimator=build, device="cuda")
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf.append_simulations(theta, x).train(training_batch_size=batch, max_num_epochs=epochs - 1,
                                               stop_after_epochs=1000)
    return 1e3 * statistics.median(inf.summary["epoch_durations_sec"][1:])


def vjp_ms(R=4096, reps=50):
    """The VJP on the 10-d context the flow sees behind the FC embedding."""
    theta, x = data(R)
    x = x[:, :10].contiguous()
    torch.manual_seed(0)
    est = posterior_nn("nsf")(theta, x).cuda()
    inp, ctx = theta.cuda().contiguous(), x.cuda().contiguous()
    out = {}
    assert est.vjp_cond_uses_tc(R), "model outside the wgmma VJP with the condition gradient"
    for name, want_cond, cond_tc in (("wgmma parameter-only", False, False), ("wgmma with d_gcond", True, True),
                                     ("SIMT with d_gcond", True, False)):
        n_part = L.load().sbi_b200_nsf_vjp_tc_parts(R) if cond_tc else est.vjp_parts(R, not want_cond)
        gpart = est._gpart(n_part)
        gcond = torch.empty(R, est.layout.C, device="cuda") if want_cond else None
        acc = torch.zeros(2, device="cuda")
        m = est._model(nbuf=3)
        rows = L.Rows(inp.data_ptr(), ctx.data_ptr(), None, R, 0)
        if not want_cond:
            assert est._vjp_uses_tc(R, True), "model outside the wgmma VJP"
        for _ in range(3):
            est.vjp(m, rows, R, None, -1.0 / R, None, gpart, None, gcond, acc, cond_tc=cond_tc)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            est.vjp(m, rows, R, None, -1.0 / R, None, gpart, None, gcond, acc, cond_tc=cond_tc)
        b.record()
        torch.cuda.synchronize()
        out[name] = a.elapsed_time(b) / reps
    return out


if __name__ == "__main__":
    print("card:", card())
    for batch, n in ((200, 20000), (4096, 4096 * 12)):
        t_id = epoch_ms(NPE, posterior_nn("nsf"), n, batch)
        t_fc = epoch_ms(NPE, posterior_nn("nsf", embedding_net=fc()), n, batch)
        print(f"NPE nsf, batch {batch}, {n} simulations: epoch {t_id:.1f} ms identity, {t_fc:.1f} ms FC embedding")
    for k, v in vjp_ms().items():
        print(f"NSF VJP, 4096 rows (theta 5-d, context 10-d): {k} {v:.3f} ms")
    t_id = epoch_ms(FMPE, posterior_flow_nn("mlp"), 20000, 200)
    t_fc = epoch_ms(FMPE, posterior_flow_nn("mlp", embedding_net=fc()), 20000, 200)
    print(f"FMPE, batch 200, 20000 simulations: epoch {t_id:.1f} ms identity, {t_fc:.1f} ms FC embedding")
