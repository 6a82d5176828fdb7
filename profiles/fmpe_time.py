"""FMPE training epoch time (20-d theta and x, batch 200), one CUDA graph per epoch."""
import os, sys, math, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torch.distributions import MultivariateNormal
from sbi_b200.inference import FMPE
D = 20
torch.manual_seed(0)
prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
theta = prior.sample((20000,))
x = theta + math.sqrt(0.1) * torch.randn_like(theta)
inf = FMPE(prior, device="cuda")
inf.append_simulations(theta, x).train(training_batch_size=200, max_num_epochs=4)
d = inf.summary["epoch_durations_sec"]
print(f"FMPE: epoch times {[round(v,3) for v in d]}  "
      f"val_loss {[round(v,4) for v in inf.summary['validation_loss']]}")
