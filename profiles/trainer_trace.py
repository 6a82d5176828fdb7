"""Seeded end-to-end trace of every trainer, for comparing two versions of the trainer module bit for bit.

    python profiles/trainer_trace.py --module sbi_b200.inference --out DIR      # one .pt per case
    python profiles/trainer_trace.py --compare DIR_A DIR_B                      # per-case differences

Each case trains on a seeded linear-Gaussian task for a few epochs and writes the network's state dict (the flat
parameters, and the embedding nets' parameters and buffers), the optimizer state (device Adam, or
torch.optim.Adam on the multi-round path) and the summary without the epoch durations.  The "short" cases stop
early, so the restore of the best weights runs too.

The NSF / MAF and flow-matching loss kernels sum the loss with float atomics, so the NPE, NLE and FMPE losses in
the summary can differ in the last bits between two runs of the same code; parameters and optimizer state do not."""
import argparse
import glob
import importlib
import math
import os
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def task(n, D=3, seed=0):
    from torch.distributions import MultivariateNormal
    torch.manual_seed(seed)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((n,))
    return prior, theta, theta + math.sqrt(0.1) * torch.randn_like(theta)


def fc_embedding(D=3):
    return torch.nn.Sequential(torch.nn.Linear(D, 16), torch.nn.ReLU(), torch.nn.Linear(16, 4))


def cases(m):
    from sbi_b200.flowmatching import posterior_flow_nn
    from sbi_b200.neural_nets import posterior_nn
    kw = dict(training_batch_size=200, max_num_epochs=3, stop_after_epochs=1000)
    short = dict(training_batch_size=200, max_num_epochs=25, stop_after_epochs=2)

    def fit(cls, n=4000, make=None, train=kw, resume=None, **ckw):
        """`make()` returns more constructor arguments, built after the task's seed (e.g. an embedding net)."""
        def run():
            prior, theta, x = task(n)
            t = cls(prior, device="cuda", **ckw, **(make() if make is not None else {}))
            t.append_simulations(theta, x).train(**train)
            if resume is not None:
                t.train(resume_training=True, **resume)
            return t
        return run

    def two_rounds():
        prior, theta, x = task(4000)
        t = m.NPE(prior, device="cuda")
        t.append_simulations(theta, x).train(**kw)
        proposal = t.build_posterior().set_default_x(x[:1])
        th2 = proposal.sample((2000,)).cpu()
        t.append_simulations(th2, th2 + math.sqrt(0.1) * torch.randn_like(th2), proposal=proposal).train(**kw)
        return t

    calib = dict(kw, calibration_kernel=lambda x: 1.0 / (1.0 + x.pow(2).sum(1)))
    nsf_embed = lambda: dict(density_estimator=posterior_nn("nsf", embedding_net=fc_embedding()))         # noqa: E731
    fm_embed = lambda: dict(density_estimator=posterior_flow_nn("mlp", embedding_net=fc_embedding()))     # noqa: E731
    return {
        "npe_nsf_tc_val": fit(m.NPE, n=20000),
        "npe_nsf_embed": fit(m.NPE, make=nsf_embed),
        "npe_maf": fit(m.NPE, density_estimator="maf"),
        "npe_calibration": fit(m.NPE, train=calib),
        "npe_short": fit(m.NPE, train=short),
        "npe_resume": fit(m.NPE, resume=dict(training_batch_size=200, max_num_epochs=5, stop_after_epochs=1000)),
        "npe_two_rounds": two_rounds,
        "nle": fit(m.NLE),
        "nle_maf": fit(m.NLE, density_estimator="maf"),
        "nle_short": fit(m.NLE, train=short),
        "nreb_resnet": fit(m.NRE_B),
        "nreb_resnet_b5000": fit(m.NRE_B, n=20000, train=dict(kw, training_batch_size=5000)),
        "nreb_mlp": fit(m.NRE_B, classifier="mlp"),
        "nreb_short": fit(m.NRE_B, train=dict(short, stop_after_epochs=1)),
        "nreb_resume": fit(m.NRE_B, resume=dict(training_batch_size=200, max_num_epochs=5, stop_after_epochs=1000)),
        "nrea": fit(m.NRE_A),
        "bnre": fit(m.BNRE),
        "nrec": fit(m.NRE_C),
        "fmpe": fit(m.FMPE),
        "fmpe_embed": fit(m.FMPE, make=fm_embed),
        "fmpe_noclip": fit(m.FMPE, train=dict(kw, clip_max_norm=None)),
        "fmpe_short_noclip": fit(m.FMPE, train=dict(short, clip_max_norm=None, max_num_epochs=40)),
        "npse_ve": fit(m.NPSE, sde_type="ve"),
        "npse_ve_short": fit(m.NPSE, sde_type="ve", train=dict(short, max_num_epochs=40)),
    }


def dump(t):
    if getattr(t, "_mr_opt", None) is not None:
        st = t._mr_opt.state_dict()["state"]
        opt = [v for i in sorted(st) for _, v in sorted(st[i].items())]
    else:
        opt = [t._opt_state, t._opt_step]
    summary = {k: v for k, v in t.summary.items() if k != "epoch_durations_sec"}
    state = {k: v.detach().cpu() for k, v in t._neural_net.state_dict().items()}
    return {"flat": t._neural_net.flat.data.cpu(), "state": state, "opt": [v.cpu() for v in opt], "summary": summary}


def compare(a, b):
    for f in sorted(glob.glob(os.path.join(a, "*.pt"))):
        x, y = torch.load(f), torch.load(os.path.join(b, os.path.basename(f)))
        d = (x["flat"] - y["flat"]).abs()
        same_state = x["state"].keys() == y["state"].keys() and all(torch.equal(x["state"][k], y["state"][k])
                                                                    for k in x["state"])
        same_opt = all(torch.equal(u, v) for u, v in zip(x["opt"], y["opt"]))
        sx, sy = x["summary"], y["summary"]
        same_summary = all(len(sx[k]) == len(sy[k]) and all(u == v or (u != u and v != v) for u, v in zip(sx[k], sy[k]))
                           for k in sx)
        sdiff = max((abs(u - v) / max(1.0, abs(v)) for k in sx for u, v in zip(sx[k], sy[k])
                     if u == u or v == v), default=0.0)
        same_len = all(len(sx[k]) == len(sy[k]) for k in sx)
        print(f"{os.path.basename(f)[:-3]:22s} state {'equal' if same_state else 'DIFF '} "
              f"opt {'equal' if same_opt else 'DIFF '} summary {'equal' if same_summary else 'DIFF '} "
              f"max|dflat| {d.max().item():.2e} >5e-5 {100 * (d > 5e-5).float().mean().item():.4f}% "
              f"summary rel {sdiff:.2e} epochs {sx['epochs_trained']} {'' if same_len else 'LENGTHS DIFFER'}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--module", default="sbi_b200.inference")
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        compare(*args.compare)
        sys.exit()
    m = importlib.import_module(args.module)
    os.makedirs(args.out, exist_ok=True)
    for name, run in cases(m).items():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            t = run()
        torch.save(dump(t), os.path.join(args.out, name + ".pt"))
        print(name, t.summary["epochs_trained"], flush=True)
