"""Cost of training and evaluating an NRE `resnet` classifier with a torch embedding net on x (prints the card
name and power limit).  Copies task: theta ~ N(0, I_2), x = 25 noisy copies of theta (50-d).

* NRE-B epoch time (num_atoms 10), identity embedding vs FC (50 -> 8) vs Conv1d (x as (2, 25)), at batch 200 and
  4096: the graph-captured step embeds the batch's B rows once and pairs them by index in the kernel;
* in the same process, the eager reference-style step that embeds the B x num_atoms repeated rows
  (nre_base.py:396-415) and runs the same classifier kernels through autograd, + clip + torch Adam;
* one potential call on 10^5 theta with the x_o embedding cached by set_x.
Epoch times are the median of the epochs after the first (which includes the graph capture); step and call times
are CUDA-event medians."""
import os
import statistics
import subprocess
import sys
import warnings

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sbi_b200.inference import NRE_B  # noqa: E402
from sbi_b200.potentials import ratio_estimator_based_potential  # noqa: E402
from sbi_b200.ratio import classifier_nn  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


class Conv(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv1d(2, 4, 5)
        self.fc = nn.Linear(4 * 21, 8)

    def forward(self, x):
        return self.fc(torch.relu(self.conv(x)).flatten(1))


def embedding(kind):
    torch.manual_seed(5)
    if kind == "identity":
        return nn.Identity()
    if kind == "fc":
        return nn.Sequential(nn.Linear(50, 32), nn.ReLU(), nn.Linear(32, 8))
    return Conv()


def data(n, kind, seed=0):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(n, 2, generator=g)
    x = theta.repeat(1, 25) + torch.randn(n, 50, generator=g)
    return theta, (x.reshape(-1, 2, 25) if kind == "conv" else x)


def epoch_ms(kind, n, batch, epochs=6):
    theta, x = data(n, kind)
    torch.manual_seed(0)
    inf = NRE_B(classifier=classifier_nn("resnet", embedding_net_x=embedding(kind)), device="cuda")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf.append_simulations(theta, x).train(training_batch_size=batch, max_num_epochs=epochs - 1,
                                               stop_after_epochs=1000)
    return 1e3 * statistics.median(inf.summary["epoch_durations_sec"][1:]), inf


def timed(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def eager_step_ms(est, theta, x, batch, num_atoms=10):
    """The reference's step: embed B x num_atoms repeated rows, logits, loss, backward, clip, Adam."""
    opt = torch.optim.Adam(est.parameters(), lr=5e-4)
    th, xx = theta[:batch].cuda(), x[:batch].cuda()
    B = th.shape[0]

    def step():
        opt.zero_grad()
        probs = torch.ones(B, B, device="cuda") * (1 - torch.eye(B, device="cuda")) / (B - 1)
        choices = torch.multinomial(probs, num_samples=num_atoms - 1, replacement=False)
        atomic = torch.cat((th[:, None, :], th[choices]), dim=1).reshape(B * num_atoms, -1)
        logits = est(atomic, xx.repeat_interleave(num_atoms, dim=0)).reshape(B, num_atoms)
        loss = -torch.mean(logits[:, 0] - torch.logsumexp(logits, dim=-1))
        loss.backward()
        torch.nn.utils.clip_grad_norm_(est.parameters(), 5.0)
        opt.step()
    return timed(step)


def main():
    print("card:", card())
    for batch in (200, 4096):
        n = max(30000, 12 * batch)
        for kind in ("identity", "fc", "conv"):
            ms, inf = epoch_ms(kind, n, batch)
            steps = int(0.9 * n) // batch
            theta, x = data(n, kind)
            eager = eager_step_ms(inf._neural_net, theta, x, batch)
            print(f"NRE-B batch {batch:5d} {kind:8s}: epoch {ms:8.2f} ms ({steps} steps, {ms / steps:.3f} ms/step); "
                  f"eager reference-style step {eager:.3f} ms")
    from torch.distributions import MultivariateNormal
    prior = MultivariateNormal(torch.zeros(2), torch.eye(2))
    for kind in ("identity", "fc", "conv"):
        _, inf = epoch_ms(kind, 30000, 200, epochs=2)
        _, xs = data(1, kind, seed=7)
        pot, _ = ratio_estimator_based_potential(inf._neural_net, prior, x_o=xs.cuda())
        th = torch.randn(100000, 2, device="cuda")
        print(f"potential on 1e5 theta ({kind}, x_o embedded once by set_x): "
              f"{timed(lambda: pot(th, track_gradients=False)):.3f} ms")


if __name__ == "__main__":
    main()
