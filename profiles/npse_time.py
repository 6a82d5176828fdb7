"""NPSE training throughput (linear-Gaussian dim 10, 100k sims, batch 4096; VE and VP), trainer level:
N_train * epochs / sum(epoch_durations_sec) incl. validation at 10 times."""
import math, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torch.distributions import MultivariateNormal
from sbi_b200.inference import NPSE
D, N, B = 10, 100_000, 4096
torch.manual_seed(0)
prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
theta = prior.sample((N,))
x = theta + math.sqrt(0.1) * torch.randn_like(theta)
for sde in ("ve", "vp"):
    inf = NPSE(prior, sde_type=sde, device="cuda")
    inf.append_simulations(theta, x).train(training_batch_size=B, max_num_epochs=5, stop_after_epochs=100)
    d = inf.summary["epoch_durations_sec"][1:]
    n_train = int(0.9 * N)
    steps = n_train // B
    print(f"NPSE {sde}: {n_train * len(d) / sum(d) / 1e6:.2f} M samples/s, "
          f"{1e3 * sum(d) / len(d) / steps:.3f} ms/step incl. validation, loss {inf.summary['training_loss'][-1]:.3f}")
