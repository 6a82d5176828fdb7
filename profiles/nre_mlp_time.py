"""NRE classifiers `resnet` / `mlp` / `linear` on one GPU: NRE-B epoch time (cfg5 shape of nre_time.py: 10-d theta
and x, 20 000 simulations, batch 200, 10 atoms, per-step CUDA graphs on), and logits throughput at 2^20 pairs with
one shared x (the rejection-sampling workload): the `mlp` SIMT kernel, the `resnet` SIMT and wgmma kernels, and a
plain torch.nn.Sequential with the `mlp`'s weights.  Prints the card and its power limit first."""
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torch.distributions import MultivariateNormal  # noqa: E402

from sbi_b200.inference import NRE_B  # noqa: E402
from sbi_b200.ratio import classifier_nn  # noqa: E402

assert torch.cuda.is_available(), "measures on a GPU"
smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv"],
                     capture_output=True, text=True).stdout.strip().replace("\n", " | ")
print(f"device: {torch.cuda.get_device_name()} | {smi}", flush=True)

D = 10
torch.manual_seed(0)
prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
theta = prior.sample((20000,))
x = theta + math.sqrt(0.1) * torch.randn_like(theta)
for model in ("resnet", "mlp", "linear"):
    inf = NRE_B(prior, classifier=model, device="cuda")
    inf.append_simulations(theta, x).train(training_batch_size=200, max_num_epochs=4)
    d = inf.summary["epoch_durations_sec"]
    print(f"NRE_B {model}: epoch times {[round(v, 3) for v in d]} s, "
          f"steps/epoch {18000 // 200}, val_loss {[round(v, 4) for v in inf.summary['validation_loss']]}", flush=True)


def timed(fn, n=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


R = 1 << 20
gd = torch.Generator(device="cuda").manual_seed(0)
th = torch.randn(R, D, device="cuda", generator=gd)
xo = x[:1].cuda()
mlp = classifier_nn("mlp")(theta, x).cuda()
res = classifier_nn("resnet")(theta, x).cuda()
runs = {"mlp SIMT": lambda: mlp.logits_raw(th, xo, x_shared=True)}
for tc in ("0", "1"):
    def run_res(tc=tc):
        os.environ["SBI_B200_TC"] = tc
        return res.logits_raw(th, xo, x_shared=True)
    runs[f"resnet {'wgmma' if tc == '1' else 'SIMT'}"] = run_res

# the same `mlp` in plain torch: standardisation, Sequential(Linear, LayerNorm, ReLU, Linear, LayerNorm, ReLU, Linear)
H = mlp.layout.H
seq = torch.nn.Sequential(torch.nn.Linear(2 * D, H), torch.nn.LayerNorm(H), torch.nn.ReLU(), torch.nn.Linear(H, H),
                          torch.nn.LayerNorm(H), torch.nn.ReLU(), torch.nn.Linear(H, 1)).cuda()
seq.load_state_dict({k[len("net."):]: v for k, v in mlp.state_dict().items() if k.startswith("net.")})
mt, st = mlp.embedding_net_theta[0]._mean.cuda(), mlp.embedding_net_theta[0]._std.cuda()
mx, sx = mlp.embedding_net_x[0]._mean.cuda(), mlp.embedding_net_x[0]._std.cuda()


@torch.no_grad()
def run_torch():
    u = torch.cat([(th - mt) / st, ((xo - mx) / sx).expand(R, -1)], dim=1)
    return seq(u).reshape(-1)


runs["mlp torch.nn.Sequential"] = run_torch
err = (runs["mlp SIMT"]() - run_torch()).abs().max().item()
print(f"logits, R = 2^20 pairs, shared x: mlp SIMT vs torch max |diff| = {err:.2e}", flush=True)
for name, fn in runs.items():
    ms = timed(fn)
    print(f"  {name:28s} {ms:8.3f} ms  {R / ms / 1e3:8.1f} M pairs/s", flush=True)
os.environ.pop("SBI_B200_TC", None)
