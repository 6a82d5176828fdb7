"""NRE-B training epoch time (cfg5 shape: 10-d theta and x, batch 200, 10 atoms), one CUDA graph per step."""
import os, sys, time, math, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torch.distributions import MultivariateNormal
from sbi_b200.inference import NRE_B
D = 10
torch.manual_seed(0)
prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
theta = prior.sample((20000,))
x = theta + math.sqrt(0.1) * torch.randn_like(theta)
inf = NRE_B(prior, device="cuda")
inf.append_simulations(theta, x).train(training_batch_size=200, max_num_epochs=4)
d = inf.summary["epoch_durations_sec"]
print(f"NRE_B: epoch times {[round(v,3) for v in d]}  "
      f"steps/epoch {18000//200}  val_loss {[round(v,4) for v in inf.summary['validation_loss']]}")
