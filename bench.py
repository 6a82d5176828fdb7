#!/usr/bin/env python
"""Headline benchmark: NSF-NPE training samples/s (+ posterior log_prob evals/s) on the
linear-Gaussian workload of BASELINE.json configs[1]:
    posterior_nn("nsf"), dim 10, 100 000 sims, training batch 4096, fp32, 1..8 x H100.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b200|reference]
                    [--workload cfg2|cfg3|cfg4|cfg5] [--dump-outputs DIR]

Default workload (cfg2, the headline line).  A "step" is one optimisation step (fused
forward+backward kernel -> partial-gradient reduce -> [gradient sum over the ranks] -> clip+Adam
kernel) on one batch of 4096 rows per GPU gathered from the HBM-resident simulation set.
* `value`  = rows of all ranks / device time (CUDA events, max over ranks), weak scaling
  (4096 rows per GPU); `strong` (N > 1, and the 32768-row point at N = 1) holds the SURVEY 8e
  partition: a fixed global batch (4096, and 32768) split across the ranks;
* `e2e`    = the same step through the host-buffer C-ABI call (pinned host batches, H2D / D2H
  inside the timed region; pipelined at every N);
* `trainer`= the user-level metric of BASELINE.md section 3, N_train * epochs / sum(epoch_durations_sec)
  through `sbi_b200.inference.NPE.train()` (validation included);
* `secondary` = posterior log_prob evals/s at one x_o, with its own CPU baseline.
`--impl reference` times the reference's own CPU training loop on the same workload: the UNMODIFIED
reference package (oracle/_ref, imported through oracle.ref_shim; its nflows
dependency is the oracle's port) when present, else the oracle port of that loop.
`--workload cfg3|cfg4|cfg5` print one line each for the other BASELINE configs (slice-sampling
potential evals/s, FMPE training samples/s, rejection proposals/s); they are secondary measurements
kept under profiles/.
`--dump-outputs DIR` (cfg2) writes what the last timed training step left behind -- the updated flat
parameters, their gradient and that step's loss accumulator -- as DIR/<name>.npy (float32), so that two builds
can be compared output for output on the same seeded inputs.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DIM = 10
NUM_SIMS = 100_000
BATCH = 4096
LOGPROB_ROWS = 1 << 22        # theta rows per log_prob step per GPU (168 MB > L2)
METRIC = "NSF-NPE train samples/sec + posterior log_prob evals/sec @1/2/4/8 GPU"
WORKLOAD = ("linearGaussian NPE posterior_nn('nsf') dim=10 100k sims batch=4096 (BASELINE configs[1]); "
            "step = fwd+bwd+clip+Adam on one batch")


def make_data(num_sims, dim, seed=0):
    """mini-sbibm gaussian_linear: theta ~ N(0, 0.1 I), x = theta + sqrt(0.1) eps."""
    import torch
    g = torch.Generator().manual_seed(seed)
    theta = math.sqrt(0.1) * torch.randn(num_sims, dim, generator=g)
    x = theta + math.sqrt(0.1) * torch.randn(num_sims, dim, generator=g)
    return theta, x


def env_world():
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")),
            int(os.environ.get("LOCAL_RANK", "0")))


# ------------------------------------------------------------------------------------ clocks
class ClockSampler:
    """Samples SM clock + throttle reasons via NVML while the timed regions run."""

    def __init__(self, index=0, period=0.02):
        self.period, self.index = period, index
        self.samples, self.reasons, self.max_mhz = [], set(), None
        self._stop = threading.Event()
        self._t = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.max_mhz = pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM)
        except Exception:
            self.nv = None

    def _loop(self):
        nv = self.nv
        names = {
            "hw_slowdown": getattr(nv, "nvmlClocksEventReasonHwSlowdown", 0x8),
            "hw_thermal_slowdown": getattr(nv, "nvmlClocksEventReasonHwThermalSlowdown", 0x40),
            "sw_thermal_slowdown": getattr(nv, "nvmlClocksEventReasonSwThermalSlowdown", 0x20),
            "sw_power_cap": getattr(nv, "nvmlClocksEventReasonSwPowerCap", 0x4),
        }
        while not self._stop.is_set():
            try:
                util = nv.nvmlDeviceGetUtilizationRates(self.h).gpu
                mhz = nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM)
                try:
                    r = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
                except Exception:
                    r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
                self.samples.append((mhz, util))
                for k, bit in names.items():
                    if r & bit:
                        self.reasons.add(k)
            except Exception:
                pass
            time.sleep(self.period)

    def start(self):
        if self.nv is not None:
            self._t = threading.Thread(target=self._loop, daemon=True)
            self._t.start()
        return self

    def stop(self):
        self._stop.set()
        if self._t is not None:
            self._t.join(timeout=1)
        loaded = sorted(m for m, u in self.samples if u > 0) or sorted(m for m, _ in self.samples)
        med = loaded[len(loaded) // 2] if loaded else None
        return {"sm_mhz": med, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons),
                "samples": len(self.samples)}


# ------------------------------------------------------------------------------------ CPU arms
def _pick_threads():
    """Intra-op thread count for the CPU arms: best of a quick probe over {16, 32, 64, all cores} on
    two optimisation steps of the port (the tiny ATen ops of this path get slower with too many
    threads).  Returns (threads, host cores)."""
    import torch
    cores = os.cpu_count() or 1
    best = None
    for c in sorted({min(c, cores) for c in (16, 32, 64, cores)}):
        _, sec, _, _ = cpu_port_train(steps=1, warmup=1, threads=c)
        if best is None or sec < best[0]:
            best = (sec, c)
    torch.set_num_threads(best[1])
    return best[1], cores


def cpu_port_train(steps, warmup, max_seconds=None, threads=None):
    """The reference's CPU training step restated (oracle port of sbi's loop on the nflows port):
    DataLoader(SubsetRandomSampler, drop_last) batch of 4096 -> loss -> backward ->
    clip_grad_norm_(5) -> Adam.  Returns (samples/s, seconds per step, threads, steps done)."""
    import torch
    from torch.nn.utils.clip_grad import clip_grad_norm_
    from oracle import sbi_port
    if threads is not None:
        torch.set_num_threads(threads)
    theta, x = make_data(NUM_SIMS, DIM)
    torch.manual_seed(0)
    tr = sbi_port.ReferenceTrainer(sbi_port.build_nsf)
    train_loader, _ = tr.get_dataloaders(theta, x, training_batch_size=BATCH)
    net = sbi_port.build_nsf(theta[tr.train_indices], x[tr.train_indices])
    tr.net = net
    opt = torch.optim.Adam(list(net.parameters()), lr=5e-4)
    it = [iter(train_loader)]

    def one_step():
        t0 = time.perf_counter()
        try:
            batch = next(it[0])
        except StopIteration:
            it[0] = iter(train_loader)
            batch = next(it[0])
        opt.zero_grad()
        losses = tr._losses(batch)
        loss = torch.mean(losses)
        losses.sum().item()
        loss.backward()
        clip_grad_norm_(net.parameters(), max_norm=5.0)
        opt.step()
        return time.perf_counter() - t0

    done, t_timed = 0, 0.0
    t_begin = time.perf_counter()
    for i in range(warmup + steps):
        dt = one_step()
        if i >= warmup:
            done += 1
            t_timed += dt
        if max_seconds is not None and time.perf_counter() - t_begin > max_seconds and done >= 2:
            break
    return done * BATCH / t_timed, t_timed / done, torch.get_num_threads(), done


def cpu_reference_train(steps, warmup, threads):
    """The UNMODIFIED reference's loop: sbi.inference.NPE(posterior_nn('nsf')).train(batch 4096) on the
    CPU (trainers/base.py:1060-1225: DataLoader, _train_epoch, _validate_epoch, _converged), imported
    through oracle.ref_shim.  `_train_epoch` is wrapped with a timer (instrumentation only).
    Returns dict(step-only samples/s, ms/step, user-level samples/s incl. validation, steps, epochs)."""
    import warnings
    import torch
    from torch.distributions import MultivariateNormal
    from oracle import ref_shim
    assert ref_shim.install()
    from sbi.inference import NPE
    from sbi.neural_nets import posterior_nn
    torch.set_num_threads(threads)
    theta, x = make_data(NUM_SIMS, DIM)
    n_train = int(0.9 * NUM_SIMS)
    spe = n_train // BATCH                                    # 21 steps per epoch (drop_last)
    warm_ep = max(1, math.ceil(warmup / spe))
    epochs = warm_ep + max(1, math.ceil(steps / spe))
    prior = MultivariateNormal(torch.zeros(DIM), 0.1 * torch.eye(DIM))
    torch.manual_seed(0)
    # the reference trainer writes TensorBoard logs under ./sbi-logs: run it from a temporary directory
    # so that the benchmark writes nothing into the (possibly read-only) tree
    cwd = os.getcwd()
    with warnings.catch_warnings(), tempfile.TemporaryDirectory(prefix="sbi_bench_") as tmp:
        warnings.simplefilter("ignore")
        os.chdir(tmp)
        try:
            inf = NPE(prior, density_estimator=posterior_nn("nsf"), device="cpu", show_progress_bars=False)
            t_train = []
            orig = inf._train_epoch

            def timed(*a, **k):
                t0 = time.perf_counter()
                out = orig(*a, **k)
                t_train.append(time.perf_counter() - t0)
                return out

            inf._train_epoch = timed
            inf.append_simulations(theta, x).train(training_batch_size=BATCH, max_num_epochs=epochs - 1,
                                                   stop_after_epochs=10 ** 6)
        finally:
            os.chdir(cwd)
    dur = inf._summary["epoch_durations_sec"]
    e = len(dur) - warm_ep
    step_s = sum(t_train[warm_ep:]) / (e * spe)
    return {"step_sps": BATCH / step_s, "ms_per_step": step_s * 1e3, "steps": e * spe, "epochs": e,
            "trainer_sps": n_train * e / sum(dur[warm_ep:]), "epoch_durations_sec": dur[warm_ep:]}


def cpu_logprob_baseline(threads, max_seconds=15.0):
    """posterior.log_prob(theta, x=x_o, norm_posterior=False) on the CPU in chunks (SURVEY 8d): the
    unmodified reference's DirectPosterior when present, else the port's flow.  Bounded sample."""
    import warnings
    import torch
    from torch.distributions import MultivariateNormal
    from oracle import ref_shim
    torch.set_num_threads(threads)
    theta, x = make_data(20_000, DIM)
    prior = MultivariateNormal(torch.zeros(DIM), 0.1 * torch.eye(DIM))
    x_o = x[:1]
    chunk = 1 << 17
    th = math.sqrt(0.1) * torch.randn(chunk, DIM)
    torch.manual_seed(0)
    if ref_shim.install():
        from sbi.inference.posteriors import DirectPosterior
        from sbi.neural_nets import posterior_nn
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            post = DirectPosterior(posterior_nn("nsf")(theta, x), prior)
        kind = "reference"

        def call():
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                return post.log_prob(th, x=x_o, norm_posterior=False)
    else:
        from oracle import sbi_port
        flow = sbi_port.build_nsf(theta, x)
        kind = "port"

        def call():
            with torch.no_grad():
                return flow.log_prob(th.unsqueeze(1), x_o)
    call()
    n, t0 = 0, time.perf_counter()
    while True:
        call()
        n += 1
        if time.perf_counter() - t0 > max_seconds or n >= 20:
            break
    sec = (time.perf_counter() - t0) / n
    return {"value": chunk / sec, "unit": "evals/s", "cores": threads, "host_cores": os.cpu_count(), "kind": kind,
            "sample": f"{n} calls of posterior.log_prob on {chunk} theta rows at one x_o (norm_posterior=False), "
                      f"{sec * 1e3:.0f} ms per call"}


def run_reference(args):
    rank, _, _ = env_world()
    if rank != 0:
        return
    if args.workload != "cfg2":
        print(json.dumps({"impl": "reference", "unavailable": f"the reference arm times cfg2 only (asked: {args.workload})"}))
        return
    from oracle import ref_shim
    threads, cores = _pick_threads()
    if ref_shim.available():
        r = cpu_reference_train(args.steps, max(args.warmup, 1), threads)
        sps, ms, done, kind = r["step_sps"], r["ms_per_step"], r["steps"], "reference"
        sample = (f"{r['epochs']} epochs x 21 optimisation steps of 4096 rows of the unmodified reference trainer "
                  f"(sbi.inference.NPE.train on oracle/nflows_port); value = rows / time inside _train_epoch "
                  f"(DataLoader collation included); user-level incl. validation: {r['trainer_sps']:.0f} samples/s")
        trainer = {"value": r["trainer_sps"], "unit": "samples/s", "epochs": r["epochs"],
                   "definition": "N_train * epochs / sum(summary['epoch_durations_sec']) (BASELINE.md section 3)"}
    else:
        sps, sec, _, done = cpu_port_train(args.steps, max(args.warmup, 1), threads=threads)
        ms, kind, trainer = sec * 1e3, "port", None
        sample = f"{done} optimisation steps of 4096 rows incl. DataLoader collation (oracle port of the loop)"
    line = {
        "impl": "reference", "metric": METRIC, "value": sps, "unit": "samples/s",
        "n_gpus": args.gpus, "steps": done, "warmup": args.warmup, "ms_per_step": ms,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
        "data": "synthetic",
        "config": {"workload": WORKLOAD, "global_batch": BATCH, "device": "cpu"},
        "cpu_baseline": {"value": sps, "unit": "samples/s", "cores": threads, "host_cores": cores, "kind": kind,
                         "sample": sample},
        "trainer": trainer,
        "e2e": {"value": sps, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))


# ------------------------------------------------------------------------------------ b200 arm
class _Ctx:
    """Process-wide setup shared by the workloads."""

    def __init__(self):
        import torch
        import torch.distributed as dist
        from sbi_b200 import _lib as L
        from sbi_b200 import build as _build
        self.rank, self.world, self.local = env_world()
        if not torch.cuda.is_available():
            raise RuntimeError("bench.py needs a GPU (no CPU fallback); use --impl reference for the CPU arm")
        torch.cuda.set_device(self.local)
        self.dev = f"cuda:{self.local}"
        if self.world > 1:
            dist.init_process_group("nccl", device_id=torch.device(self.dev))
        _build.build()
        self.lib = L.load()
        self.L, self.torch, self.dist = L, torch, dist

    def barrier(self):
        if self.world > 1:
            self.dist.barrier()
        self.torch.cuda.synchronize()

    def max_over_ranks(self, v):
        t = self.torch.tensor([float(v)], device=self.dev)
        if self.world > 1:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return float(t.item())

    def finish(self):
        if self.world > 1:
            self.dist.destroy_process_group()


class StepRunner:
    """One optimisation step of `rows` rows per rank on device-resident data, captured in CUDA graphs
    (one per index slot).  upstream gradient -1/(rows * world): the ranks' rows form one global batch."""

    def __init__(self, cx, est, theta_d, x_d, n_train, rows, peer, state=None):
        torch, L, lib = cx.torch, cx.L, cx.lib
        self.cx, self.est, self.rows, self.peer = cx, est, rows, peer
        self.theta_d, self.x_d = theta_d, x_d
        P = est.layout.n_params
        self.P = P
        dev = cx.dev
        self.n_part = est.vjp_parts(rows)          # tensor-core step: one slab per 128-row tile
        self.gpart = torch.zeros(self.n_part, P, device=dev)
        self.grad = torch.zeros(P, device=dev)
        self.grad_local = torch.zeros(P, device=dev) if peer is not None else self.grad
        self.state = torch.zeros(2 * P, device=dev) if state is None else state
        self.step_ctr = torch.zeros(2, dtype=torch.int32, device=dev)
        self.loss_acc = torch.zeros(2, device=dev)
        self.sumsq = torch.zeros(max(lib.sbi_b200_sumsq_blocks(P), lib.sbi_b200_peer_blocks(P)), device=dev)
        self.mask = est.net._mask
        self.idx_pool = torch.stack([torch.randperm(n_train, device=dev)[:rows] for _ in range(16)])
        self.graphs = None
        # kernels per step: [operand pack + forward + backward | SIMT vjp] + reduce [+ peer sum] + clip/Adam
        self.launches_per_step = (3 if est._vjp_uses_tc(rows, True) else 1) + (3 if peer is not None else 2)

    def step(self, i):
        cx, L, lib, est, P = self.cx, self.cx.L, self.cx.lib, self.est, self.P
        world = cx.world
        m = est._model(nbuf=3)
        idx = self.idx_pool[i % self.idx_pool.shape[0]]
        rows = L.Rows(self.theta_d.data_ptr(), self.x_d.data_ptr(), idx.data_ptr(), self.rows, 0)
        est.vjp(m, rows, self.rows, None, -1.0 / (self.rows * world), None, self.gpart, None, None, self.loss_acc)
        if self.peer is not None:
            L.check(lib.sbi_b200_reduce_partials(L.ptr(self.gpart), self.n_part, P, L.ptr(self.grad_local),
                                                 L.stream_ptr()), "reduce")
            self.peer.sum(self.grad_local, self.grad, self.mask, self.sumsq)
            L.check(lib.sbi_b200_adam_clip_step_norm(L.ptr(est.flat.data), L.ptr(self.grad), L.ptr(self.state),
                                                     L.ptr(self.step_ctr), L.ptr(self.mask), P, 5e-4, 0.9, 0.999,
                                                     1e-8, 5.0, 1.0, L.ptr(self.sumsq), self.peer.n_sumsq,
                                                     L.stream_ptr()), "adam")
        elif world > 1:
            L.check(lib.sbi_b200_reduce_partials(L.ptr(self.gpart), self.n_part, P, L.ptr(self.grad),
                                                 L.stream_ptr()), "reduce")
            cx.dist.all_reduce(self.grad)
            L.check(lib.sbi_b200_adam_clip_step(L.ptr(est.flat.data), L.ptr(self.grad), L.ptr(self.state),
                                                L.ptr(self.step_ctr), L.ptr(self.mask), P, 5e-4, 0.9, 0.999, 1e-8,
                                                5.0, 1.0, L.stream_ptr()), "adam")
        else:
            L.check(lib.sbi_b200_reduce_partials_norm(L.ptr(self.gpart), self.n_part, P, L.ptr(self.grad),
                                                      L.ptr(self.mask), L.ptr(self.sumsq), L.stream_ptr()), "reduce")
            L.check(lib.sbi_b200_adam_clip_step_norm(L.ptr(est.flat.data), L.ptr(self.grad), L.ptr(self.state),
                                                     L.ptr(self.step_ctr), L.ptr(self.mask), P, 5e-4, 0.9, 0.999,
                                                     1e-8, 5.0, 1.0, L.ptr(self.sumsq),
                                                     lib.sbi_b200_sumsq_blocks(P), L.stream_ptr()), "adam")

    def prepare(self, warmup):
        cx, torch = self.cx, self.cx.torch
        for i in range(warmup):
            self.step(i)
        torch.cuda.synchronize()
        if cx.world == 1 or self.peer is not None:
            if cx.world > 1:
                cx.dist.barrier()
            self.graphs = []
            for i in range(self.idx_pool.shape[0]):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self.step(i)
                self.graphs.append(g)

    def timed(self, K, flush):
        """K steps, each bracketed by CUDA events; L2 flushed (untimed) between steps.
        Returns per-step ms (this rank)."""
        cx, torch = self.cx, self.cx.torch
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
        cx.barrier()
        for i in range(K):
            flush.zero_()
            if i == K - 1:
                self.loss_acc.zero_()      # the loss accumulator then holds the last step's loss alone
            ev[i][0].record()
            if self.graphs is not None:
                self.graphs[i % len(self.graphs)].replay()
            else:
                self.step(i)
            ev[i][1].record()
        cx.barrier()
        return [a.elapsed_time(b) for a, b in ev]


def run_cfg2(args):
    cx = _Ctx()
    torch, dist, L, lib = cx.torch, cx.dist, cx.L, cx.lib
    from sbi_b200.neural_nets import posterior_nn
    rank, world, dev = cx.rank, cx.world, cx.dev
    K, W = args.steps, max(args.warmup, 3)
    theta, x = make_data(NUM_SIMS, DIM, seed=rank)          # weak scaling: every rank its own shard
    torch.manual_seed(0)
    n_train = int(0.9 * NUM_SIMS)
    est = posterior_nn("nsf")(theta[:n_train], x[:n_train]).to(dev)
    if world > 1:
        for t in list(est.parameters()) + list(est.buffers()):
            dist.broadcast(t.data, 0)
        est._cache.clear()
    lay = est.layout
    P = lay.n_params
    theta_d, x_d = theta.to(dev), x.to(dev)
    B = BATCH
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)   # > 50 MB L2
    # N > 1: the flat gradients are summed over NVLink peer memory by our own kernel (csrc/peer.cu);
    # SBI_B200_NCCL=1 keeps the NCCL all-reduce instead (no CUDA graph then)
    peer = None
    if world > 1:
        from sbi_b200.parallel import make_gradient_exchange
        peer = make_gradient_exchange(P)
    clocks = ClockSampler(index=cx.local).start()

    # ---- training: device-resident leg (value), weak scaling ------------------------------------
    run = StepRunner(cx, est, theta_d, x_d, n_train, B, peer)
    run.prepare(W)
    ms_steps = run.timed(K, flush)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, params=est.flat.data, grad=run.grad, loss_acc=run.loss_acc)
    ms_step = cx.max_over_ranks(sum(ms_steps) / K)
    train_sps = world * B / (ms_step * 1e-3)
    n_launch = K * run.launches_per_step
    # replicas must still be bit-identical after W + K data-parallel updates
    identical = None
    if world > 1:
        both = [torch.zeros_like(est.flat.data) for _ in range(world)]
        dist.all_gather(both, est.flat.data)
        identical = bool(all(torch.equal(both[0], b) for b in both))

    # ---- strong scaling (SURVEY 8e): fixed global batch split across the ranks --------------------
    strong = {}
    for gb in (4096, 32768):
        if gb % world or (world == 1 and gb == B):
            continue
        r = StepRunner(cx, est, theta_d, x_d, n_train, gb // world, peer)
        r.prepare(W)
        ks = max(5, min(K, 20))
        ms = cx.max_over_ranks(sum(r.timed(ks, flush)) / ks)
        strong[str(gb)] = {"global_batch": gb, "rows_per_gpu": gb // world, "ms_per_step": ms,
                           "samples_per_s": gb / (ms * 1e-3), "steps": ks}
        del r
    if world == 1:
        strong[str(B)] = {"global_batch": B, "rows_per_gpu": B, "ms_per_step": ms_step,
                          "samples_per_s": train_sps, "steps": K}

    # ---- dominant kernel alone (roofline): fused fwd+bwd kernel ------------------------------
    kev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
    m = est._model(nbuf=3)
    for i in range(K):
        flush.zero_()
        idx = run.idx_pool[i % run.idx_pool.shape[0]]
        rows = L.Rows(theta_d.data_ptr(), x_d.data_ptr(), idx.data_ptr(), B, 0)
        kev[i][0].record()
        est.vjp(m, rows, B, None, -1.0 / B, None, run.gpart, None, None, None)
        kev[i][1].record()
    torch.cuda.synchronize()
    vjp_ms = sum(a.elapsed_time(b) for a, b in kev) / K
    real_params = lay.num_real_params()
    alg_bytes = B * (4 * DIM + 4 * DIM + 4) + 2 * 4 * real_params   # rows in + weights in + grads out
    flops = 2.0 * B * 3 * _nsf_macs(lay)                              # fwd + 2x bwd (no recompute counted)
    peaks = _peaks()
    achieved = alg_bytes / (vjp_ms * 1e-3) / 1e9
    traffic = _traffic()
    vjp_info = _vjp_kernel_info(est, B)

    # ---- log_prob leg (secondary metric) ---------------------------------------------------------
    R = LOGPROB_ROWS
    th_eval = (math.sqrt(0.1) * torch.randn(R, DIM, device=dev))
    x_o = x_d[:1].contiguous()
    for _ in range(3):
        est._logprob_raw(th_eval, x_o, True)
    lk = max(5, min(K, 20))
    lev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(lk)]
    cx.barrier()
    for i in range(lk):
        lev[i][0].record()
        est._logprob_raw(th_eval, x_o, True)
        lev[i][1].record()
    cx.barrier()
    lp_ms = cx.max_over_ranks(sum(a.elapsed_time(b) for a, b in lev) / lk)
    lp_eps = world * R / (lp_ms * 1e-3)
    lp_bytes = R * (4 * DIM + 4)
    lp_flops = 2.0 * R * _nsf_macs(lay)
    tc_used = est._tc_state(est._model(nbuf=2)) is not None and R >= est.TC_MIN_ROWS

    # ---- end to end: host buffers through the C ABI (pipelined at every N) ------------------------
    ws = L.TrainWs()
    st_in = torch.empty(max(B, 1 << 20), DIM, device=dev)
    st_c = torch.empty(max(B, 1 << 20), DIM, device=dev)
    st_lp = torch.empty(max(B, 1 << 20), device=dev)
    ws.d_input, ws.d_cond, ws.d_logp = st_in.data_ptr(), st_c.data_ptr(), st_lp.data_ptr()
    ws.d_gpart, ws.d_grad, ws.d_state = run.gpart.data_ptr(), run.grad.data_ptr(), run.state.data_ptr()
    ws.d_step, ws.d_mask, ws.d_loss_acc = run.step_ctr.data_ptr(), run.mask.data_ptr(), run.loss_acc.data_ptr()
    ws.cap_rows = st_in.shape[0]
    ws.d_sumsq = run.sumsq.data_ptr()
    tc_keep = est._tc_train_state(est._model(nbuf=3), pack=False) if est._vjp_uses_tc(B, True) else None
    if tc_keep is not None:      # the host step runs the tensor-core forward+backward pair
        save = torch.empty(int(lib.sbi_b200_nsf_vjp_tc_save_bytes(C.byref(est._model(nbuf=3)), B)) // 4 + 1, device=dev)
        ws.tc_fwd, ws.tc_bwd, ws.tc_pack = (C.addressof(tc_keep[0]), C.addressof(tc_keep[1]), C.addressof(tc_keep[2]))
        ws.d_save, ws.save_bytes = save.data_ptr(), save.numel() * 4
    h_th2 = [torch.empty(B, DIM).pin_memory() for _ in range(2)]
    h_x2 = [torch.empty(B, DIM).pin_memory() for _ in range(2)]
    h_loss = torch.zeros(2).pin_memory()
    pipe = lib.sbi_b200_pipe_create()
    perm_host = torch.randperm(n_train)
    pctx = None
    if peer is not None:
        pctx = L.PeerCtx(C.cast(peer._ptrs, C.c_void_p), world, rank, run.grad_local.data_ptr())

    def host_step(i):
        """One optimisation step from a pinned host batch through the pipelined C-ABI entry: enqueue
        step i (H2D + kernels [+ peer-memory gradient sum] + D2H), get step i-1's loss back."""
        idx = perm_host[(i * B) % (n_train - B):][:B]
        mm = est._model(nbuf=3)
        a, b = h_th2[i & 1], h_x2[i & 1]
        torch.index_select(theta, 0, idx, out=a)      # host batch assembly (the reference's
        torch.index_select(x, 0, idx, out=b)          # DataLoader collation)
        if world == 1:
            L.check(lib.sbi_b200_nsf_train_step_host_async(
                C.byref(mm), C.byref(ws), pipe, a.data_ptr(), b.data_ptr(), B, 5e-4, 0.9, 0.999, 1e-8,
                5.0, h_loss.data_ptr(), L.stream_ptr()), "train_step_host_async")
        elif pctx is not None:
            L.check(lib.sbi_b200_nsf_train_step_host_async_dp(
                C.byref(mm), C.byref(ws), pipe, C.byref(pctx), a.data_ptr(), b.data_ptr(), B, 5e-4, 0.9, 0.999,
                1e-8, 5.0, h_loss.data_ptr(), L.stream_ptr()), "train_step_host_async_dp")
        else:       # NCCL fallback: blocking pieces
            st_in[:B].copy_(a, non_blocking=True)
            st_c[:B].copy_(b, non_blocking=True)
            run.loss_acc.zero_()
            rows = L.Rows(st_in.data_ptr(), st_c.data_ptr(), None, B, 0)
            est.vjp(mm, rows, B, None, -1.0 / (B * world), None, run.gpart, None, None, run.loss_acc)
            L.check(lib.sbi_b200_reduce_partials(L.ptr(run.gpart), run.n_part, P, L.ptr(run.grad), L.stream_ptr()), "reduce")
            dist.all_reduce(run.grad)
            L.check(lib.sbi_b200_adam_clip_step(L.ptr(est.flat.data), L.ptr(run.grad), L.ptr(run.state),
                                                L.ptr(run.step_ctr), L.ptr(run.mask), P, 5e-4, 0.9, 0.999, 1e-8, 5.0,
                                                1.0, L.stream_ptr()), "adam")
            h_loss.copy_(run.loss_acc, non_blocking=True)
            torch.cuda.current_stream().synchronize()

    torch.set_num_threads(min(8, os.cpu_count() or 1))   # host-side gathers are tiny: avoid a 128-thread fork/join
    for i in range(W):
        host_step(i)
    lib.sbi_b200_pipe_drain(pipe, h_loss.data_ptr())
    cx.barrier()
    t0 = time.perf_counter()
    for i in range(K):
        host_step(W + i)
    lib.sbi_b200_pipe_drain(pipe, h_loss.data_ptr())   # the last step's loss is read inside the timed region
    cx.barrier()
    e2e_s = cx.max_over_ranks((time.perf_counter() - t0) / K)
    # log_prob e2e on 2^20 host rows per GPU
    Rh = 1 << 20
    h_eval = th_eval[:Rh].cpu().pin_memory()
    h_xo = x_o.cpu().pin_memory()
    h_out = torch.empty(Rh).pin_memory()
    mm = est._model(nbuf=2)
    tcs = est._tc_state(mm)

    def lp_host():
        if tcs is not None:
            L.check(lib.sbi_b200_nsf_logprob_host_tc(C.byref(mm), C.byref(tcs), C.byref(ws), h_eval.data_ptr(),
                                                     h_xo.data_ptr(), Rh, 1, h_out.data_ptr(), L.stream_ptr()),
                    "logprob_host_tc")
        else:
            L.check(lib.sbi_b200_nsf_logprob_host(C.byref(mm), C.byref(ws), h_eval.data_ptr(), h_xo.data_ptr(),
                                                  Rh, 1, h_out.data_ptr(), L.stream_ptr()), "logprob_host")

    for _ in range(2):
        lp_host()
    cx.barrier()
    t0 = time.perf_counter()
    for _ in range(5):
        lp_host()
    cx.barrier()
    lp_e2e_s = cx.max_over_ranks((time.perf_counter() - t0) / 5)
    e2e = {"value": world * B / e2e_s, "unit": "samples/s", "ms_per_step": e2e_s * 1e3,
           "h2d_bytes_per_step": world * B * 2 * DIM * 4, "d2h_bytes_per_step": world * 8,
           "api": ("sbi_b200_nsf_train_step_host_async" if world == 1 else
                   "sbi_b200_nsf_train_step_host_async_dp (peer-memory gradient sum inside)" if pctx is not None
                   else "host batch -> H2D -> vjp -> reduce -> NCCL all-reduce -> clip+Adam -> D2H loss, per rank")
                  + " (C ABI, pinned host batch; each step's H2D/D2H inside, result of step i read while step i+1 runs)",
           "log_prob": {"value": world * Rh / lp_e2e_s, "unit": "evals/s", "rows": world * Rh,
                        "api": "sbi_b200_nsf_logprob_host_tc" if tcs is not None else "sbi_b200_nsf_logprob_host",
                        "h2d_bytes_per_step": world * (Rh * DIM * 4 + DIM * 4), "d2h_bytes_per_step": world * Rh * 4}}
    clk = clocks.stop()
    if peer is not None:
        if peer.error():
            raise RuntimeError("peer gradient exchange timed out")
        peer.close()

    # ---- user-level trainer throughput (BASELINE.md section 3) ------------------------------------
    trainer = None
    if not args.no_trainer:
        from torch.distributions import MultivariateNormal
        from sbi_b200.inference import NPE
        prior = MultivariateNormal(torch.zeros(DIM), 0.1 * torch.eye(DIM))
        torch.manual_seed(0)
        inf = NPE(prior, density_estimator="nsf", device=dev)
        if world > 1:
            inf.data_parallel("local")
        epochs = 20
        inf.append_simulations(theta, x).train(training_batch_size=B, max_num_epochs=epochs - 1,
                                               stop_after_epochs=10 ** 6)
        dur = inf.summary["epoch_durations_sec"]
        sec = cx.max_over_ranks(sum(dur))
        trainer = {"value": world * n_train * len(dur) / sec, "unit": "samples/s", "epochs": len(dur),
                   "epoch_ms": 1e3 * sec / len(dur), "validation_loss_last": inf.summary["validation_loss"][-1],
                   "api": "sbi_b200.inference.NPE(...).append_simulations().train(training_batch_size=4096)"
                          + ("" if world == 1 else ".data_parallel('local')"),
                   "definition": "N_train * epochs / sum(summary['epoch_durations_sec']), validation included "
                                 "(BASELINE.md section 3); one CUDA graph per epoch"}

    # ---- CPU baselines (bounded samples), rank 0 at N=1 only --------------------------------------
    cpu = lp_cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        from oracle import ref_shim
        threads, cores = _pick_threads()
        if ref_shim.available():
            r = cpu_reference_train(steps=42, warmup=21, threads=threads)
            cpu = {"value": r["step_sps"], "unit": "samples/s", "cores": threads, "host_cores": cores,
                   "kind": "reference",
                   "sample": f"{r['steps']} optimisation steps of 4096 rows of the unmodified reference trainer on the "
                             f"nflows port (time inside _train_epoch, {r['ms_per_step']:.0f} ms/step); user-level incl. "
                             f"validation {r['trainer_sps']:.0f} samples/s"}
        else:
            sps, sec, _, done = cpu_port_train(steps=40, warmup=2, max_seconds=20, threads=threads)
            cpu = {"value": sps, "unit": "samples/s", "cores": threads, "host_cores": cores, "kind": "port",
                   "sample": f"{done} optimisation steps of 4096 rows (oracle port of the reference loop incl. "
                             f"DataLoader collation), {sec * 1e3:.0f} ms/step"}
        lp_cpu = cpu_logprob_baseline(threads)

    if rank == 0:
        line = {
            "metric": METRIC, "value": train_sps, "unit": "samples/s", "n_gpus": world, "steps": K,
            "warmup": W, "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": WORKLOAD,
                       "global_batch": B * world, "per_gpu_batch": B, "params": real_params,
                       "parallelism": f"dp{world}", "l2": "flushed between timed steps (256 MiB memset, untimed)",
                       "launch": "cuda-graph per step" if run.graphs is not None else "eager",
                       "gradient_exchange": ("none" if world == 1 else
                                             "peer-memory sum kernel over NVLink (csrc/peer.cu)" if peer is not None
                                             else "NCCL all-reduce")},
            "roofline": {"bound": "hbm", "kernel": vjp_info["kernel"], "achieved": achieved,
                         "peak": peaks["hbm_gbs"], "unit": "GB/s", "frac": achieved / peaks["hbm_gbs"],
                         "traffic": traffic.get(vjp_info["traffic_key"], {}).get("dram_bytes_per_launch"),
                         "traffic_source": traffic.get("_source", "profiles/ (ncu --set full, B=4096)"),
                         "peak_source": peaks["source"],
                         "alg_bytes_per_launch": alg_bytes, "kernel_ms": vjp_ms,
                         "compute": {"achieved_tflops": flops / (vjp_ms * 1e-3) / 1e12,
                                     "fp32_fma_nominal_tflops": 67.0,
                                     "tf32_tensor_peak_tflops": peaks["bf16_tflops"] / 2.0,
                                     "note": "the fused kernel is compute/latency bound (SURVEY 8d): algorithmic "
                                             "flops = 2 x 3 x conditioner MACs per row (fwd + dX + dW)"}},
            "secondary": {"metric": "posterior log_prob evals/sec", "value": lp_eps, "unit": "evals/s",
                          "rows_per_step_per_gpu": R, "ms_per_step": lp_ms,
                          "l2": "inputs (168 MB) larger than L2",
                          "roofline": _lp_roofline(tc_used, lp_bytes, lp_flops, lp_ms, peaks),
                          "cpu_baseline": lp_cpu},
            "strong": strong, "replicas_bit_identical": identical, "trainer": trainer,
            "cpu_baseline": cpu, "clocks": clk, "e2e": e2e, "gpu_launches": n_launch,
            "step_ms_minmax": [min(ms_steps), max(ms_steps)],
        }
        print(json.dumps(line))
    cx.finish()


def dump_outputs(out_dir, **arrays):
    """Write each array as out_dir/<name>.npy in float32."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for name, t in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), t.detach().float().cpu().numpy())


def _vjp_kernel_info(est=None, B=BATCH):
    """Which VJP kernels the library dispatches to at B rows (names for the roofline entry)."""
    if est is not None and est._vjp_uses_tc(B, True):
        return {"kernel": "nsf_logprob_tc_kernel<50,10,false,SAVE> + nsf_vjp_tc_kernel<50,10> (wgmma forward + "
                          "backward pair; operand re-pack included in the timing)",
                "traffic_key": "nsf_vjp_tc", "tc": True}
    return {"kernel": "nsf_vjp_kernel<32,2,2,true>", "traffic_key": "nsf_vjp_kernel", "tc": False}


def _lp_roofline(tc_used, lp_bytes, lp_flops, lp_ms, peaks):
    """Roofline entry of the log_prob kernel.  Tensor-core path: algorithmic fp32-equivalent flops
    (2 x MACs of the linears, no padding, counted once although 3xTF32 issues three MMAs per
    product) against the tf32 tensor peak, taken as half the measured dense bf16 peak."""
    sec = lp_ms * 1e-3
    if not tc_used:
        return {"bound": "hbm", "kernel": "nsf_logprob_kernel<64,4>", "achieved": lp_bytes / sec / 1e9,
                "peak": peaks["hbm_gbs"], "unit": "GB/s", "frac": lp_bytes / sec / 1e9 / peaks["hbm_gbs"],
                "fp32_fma_tflops": lp_flops / sec / 1e12}
    peak = peaks["bf16_tflops"] / 2.0
    ach = lp_flops / sec / 1e12
    return {"bound": "tensor", "kernel": "nsf_logprob_tc_kernel<50,10,false>", "achieved": ach, "peak": peak,
            "unit": "TFLOP/s", "frac": ach / peak,
            "peak_source": peaks["source"] + "; tf32 = bf16/2",
            "note": "3xTF32: the tensor pipe executes 3x the algorithmic flops (plus K/N padding 50->56/64)",
            "hbm_gbs": lp_bytes / sec / 1e9}


def _nsf_macs(lay):
    """Multiply-accumulates per row of one forward pass (conditioners + LU; spline excluded)."""
    tot = 0
    for l in range(lay.T):
        n_id, n_tr = len(lay.id_feats[l]), len(lay.tr_feats[l])
        tot += (n_id + lay.C) * lay.H + lay.NB * (2 * lay.H * lay.H + lay.C * lay.H)
        tot += lay.H * n_tr * lay.NPAR + lay.D * lay.D
    return tot


def _traffic():
    for name in ("r02_traffic.json", "r01_traffic.json"):
        p = os.path.join(ROOT, "profiles", name)
        try:
            d = json.load(open(p))
            d.setdefault("_source", f"profiles/{name} (ncu --set full, B=4096)")
            return d
        except Exception:
            continue
    return {}


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d.get("bf16_tflops", 989.0),
                "source": "MEASURED_PEAKS.json (measured)"}
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "source": "H100 SXM data sheet (dense, 700 W), not measured"}


# ------------------------------------------------------------------------------------ other BASELINE configs
def _line(cx, metric, value, unit, ms, K, W, config, extra):
    d = {"metric": metric, "value": value, "unit": unit, "n_gpus": cx.world, "steps": K, "warmup": W,
         "ms_per_step": ms, "higher_is_better": True, "scaling": extra.pop("scaling", "weak"), "vs_baseline": None,
         "dtype": "f32", "data": "synthetic", "config": config}
    d.update(extra)
    return d


def run_cfg4(args):
    """BASELINE configs[3]: FMPE, dim 20, 1M sims, batch 16384 (global), data parallel.  Trainer-level:
    N_train * epochs / sum(epoch_durations_sec) through sbi_b200.inference.FMPE.train() (validation at 10
    times included), partition='global' (the 16384-row batch is split over the ranks)."""
    cx = _Ctx()
    torch = cx.torch
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import FMPE
    D, N, B = 20, 1_000_000, 16384
    theta, x = make_data(N, D, seed=0)                        # identical on every rank (global partition)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    clocks = ClockSampler(index=cx.local).start()
    torch.manual_seed(0)
    inf = FMPE(prior, device=cx.dev)
    if cx.world > 1:
        inf.data_parallel("global")
    # the trainer runs whole epochs of 54 steps: --steps is rounded up to whole epochs (the first, untimed
    # epoch comes on top)
    epochs = max(1, math.ceil(args.steps / 54))
    inf.append_simulations(theta, x).train(training_batch_size=B, max_num_epochs=epochs, stop_after_epochs=10 ** 6)
    dur = inf.summary["epoch_durations_sec"][1:]
    sec = cx.max_over_ranks(sum(dur))
    n_train = int(0.9 * N)
    steps = (n_train // B) * len(dur)
    cpu = None
    if cx.rank == 0 and cx.world == 1 and not args.no_cpu_baseline:
        cpu = _cpu_fm_baseline(D, B)
    if cx.rank == 0:
        print(json.dumps(_line(
            cx, "FMPE train samples/sec (trainer-level, validation included)", n_train * len(dur) / sec, "samples/s",
            1e3 * sec / steps, steps, 54,
            {"workload": "linearGaussian FMPE posterior_flow_nn('mlp') dim=20 1M sims batch=16384 (BASELINE configs[3])",
             "global_batch": B, "parallelism": f"dp{cx.world} partition=global",
             "api": "sbi_b200.inference.FMPE.train()"},
            {"scaling": "strong", "epochs": len(dur), "epoch_ms": 1e3 * sec / len(dur), "cpu_baseline": cpu,
             "training_loss": inf.summary["training_loss"][-1], "clocks": clocks.stop(),
             "gpu_launches": steps * (4 if cx.world > 1 else 3) + 10 * len(dur)})))
    cx.finish()


def _cpu_fm_baseline(D, B, max_seconds=15.0):
    """The reference's FMPE optimisation step on the CPU (oracle port of FlowMatchingEstimator.loss +
    Adam + clipping), bounded sample."""
    import torch
    from torch.nn.utils.clip_grad import clip_grad_norm_
    from oracle import sbi_port
    threads = min(32, os.cpu_count() or 1)
    torch.set_num_threads(threads)
    theta, x = make_data(4 * B, D)
    net = sbi_port.build_flow_matching_estimator(theta, x)
    opt = torch.optim.Adam(net.parameters(), lr=5e-4)
    n, t0 = 0, None
    while True:
        i = (n * B) % (3 * B)
        opt.zero_grad()
        net.loss(theta[i:i + B], x[i:i + B]).mean().backward()
        clip_grad_norm_(net.parameters(), 5.0)
        opt.step()
        if t0 is None:
            t0 = time.perf_counter()      # first step = warm-up
            continue
        n += 1
        if time.perf_counter() - t0 > max_seconds or n >= 30:
            break
    sec = (time.perf_counter() - t0) / n
    return {"value": B / sec, "unit": "samples/s", "cores": threads, "host_cores": os.cpu_count(), "kind": "port",
            "sample": f"{n} optimisation steps of {B} rows (loss + backward + clip + Adam, no DataLoader), "
                      f"{sec * 1e3:.0f} ms/step"}


def run_cfg5(args):
    """BASELINE configs[4]: NRE-B resnet classifier, dim 10; 1M rejection proposals sharded over the
    ranks (parallel.rejection_fixed_budget: same seeded candidate / uniform streams on every rank, each
    rank evaluates its block with the tensor-core ratio kernel, all-gather of (index, row))."""
    cx = _Ctx()
    torch = cx.torch
    from torch.distributions import MultivariateNormal
    from sbi_b200 import parallel
    from sbi_b200.inference import NRE_B
    from sbi_b200.potentials import ratio_estimator_based_potential
    D, N = 10, 200_000
    theta, x = make_data(N, D, seed=0)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    clocks = ClockSampler(index=cx.local).start()
    torch.manual_seed(0)
    inf = NRE_B(prior, classifier="resnet", device=cx.dev)
    if cx.world > 1:
        inf.data_parallel("global")
    epochs = 3
    inf.append_simulations(theta, x).train(training_batch_size=200 if cx.world == 1 else 200 * cx.world,
                                           max_num_epochs=epochs - 1, stop_after_epochs=10 ** 6)
    dur = inf.summary["epoch_durations_sec"][1:]
    train_sec = cx.max_over_ranks(sum(dur))
    est = inf._neural_net
    pot, _ = ratio_estimator_based_potential(est, prior, x_o=x[:1])
    from sbi_b200.posteriors import prior_to_device
    prior_d = prior_to_device(prior, cx.dev)      # log_prob as one matmul instead of torch's triangular solve
    chol = math.sqrt(0.1)
    NP = 1_000_000

    def proposal_sample(n, gen):
        return chol * torch.randn(n, D, generator=gen)

    # bound = max over the proposals (found once, as rejection_sample's search would) + log m
    with torch.no_grad():
        probe = proposal_sample(1 << 16, torch.Generator().manual_seed(7)).to(cx.dev)
        log_bound = float((pot(probe, track_gradients=False) - prior_d.log_prob(probe)).max()) + math.log(1.2)
    t = torch.tensor([log_bound], device=cx.dev)
    if cx.world > 1:
        cx.dist.broadcast(t, 0)
    log_bound = float(t.item())
    K = max(1, args.steps)
    times, n_acc = [], None
    for i in range(3 + K):
        cx.barrier()
        t0 = time.perf_counter()
        rows, idx = parallel.rejection_fixed_budget(lambda th: pot(th, track_gradients=False), proposal_sample,
                                                    prior_d.log_prob, log_bound, NP, seed=100 + i, device=cx.dev)
        cx.barrier()
        if i >= 3:
            times.append(time.perf_counter() - t0)
        n_acc = int(idx.shape[0])
    sec = cx.max_over_ranks(sum(times) / len(times))
    # potential-only device time (the sharded part)
    lo, hi = parallel.shard_range(NP, cx.rank, cx.world)
    mine = proposal_sample(NP, torch.Generator().manual_seed(1))[lo:hi].to(cx.dev)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
    cx.barrier()
    for a, b in ev:
        a.record()
        pot(mine, track_gradients=False)
        b.record()
    cx.barrier()
    pot_ms = cx.max_over_ranks(sum(a.elapsed_time(b) for a, b in ev) / K)
    if cx.rank == 0:
        n_train = int(0.9 * N)
        print(json.dumps(_line(
            cx, "rejection proposals/sec (NRE-B resnet potential, 1M prior proposals, fixed budget)", NP / sec,
            "proposals/s", sec * 1e3, K, 3,
            {"workload": "SNRE-B classifier_nn('resnet') dim=10 200k sims; rejection sampler 1M proposals "
                         "(BASELINE configs[4])", "parallelism": f"proposals sharded over {cx.world} ranks",
             "api": "sbi_b200.parallel.rejection_fixed_budget"},
            {"scaling": "strong", "accepted": n_acc,
             "potential_only": {"ms": pot_ms, "proposals_per_s": NP / (pot_ms * 1e-3),
                                "note": "ratio_forward_tc kernel + prior log-prob on this rank's block, device time"},
             "note": "the whole-call time includes generating the seeded CPU candidate / uniform streams "
                     "(reference semantics, rejection.py:170-200) and their H2D copy",
             "nre_training": {"samples_per_s": n_train * len(dur) / train_sec, "epochs": len(dur),
                              "batch": 200 if cx.world == 1 else 200 * cx.world,
                              "api": "sbi_b200.inference.NRE_B.train(num_atoms=10)"},
             "clocks": clocks.stop(), "gpu_launches": K})))
    cx.finish()


def run_cfg3(args):
    """BASELINE configs[2]: two-moons NLE nsf, slice_np_vectorized with 1000 chains, 10 000 samples after
    200 warm-up sweeps.  Reports potential evaluations/s and samples/s of posterior.sample()."""
    cx = _Ctx()
    torch = cx.torch
    from torch.distributions import Independent, Uniform
    from sbi_b200.inference import NLE
    from tests.helpers import two_moons_simulator
    torch.manual_seed(0)
    prior = Independent(Uniform(-torch.ones(2), torch.ones(2)), 1)
    theta = prior.sample((50_000,))
    x = two_moons_simulator(theta)
    clocks = ClockSampler(index=cx.local).start()
    nle = NLE(prior, density_estimator="nsf", device=cx.dev)
    nle.append_simulations(theta, x).train(training_batch_size=1000, max_num_epochs=30)
    dur = nle.summary["epoch_durations_sec"]
    x_o = torch.tensor([[0.0, 0.0]])
    chains = 1000 // cx.world
    post = nle.build_posterior(mcmc_method="slice_np_vectorized",
                               mcmc_parameters=dict(num_chains=chains, warmup_steps=200, thin=1))
    post.sample((1000,), x=x_o)
    times, evals, steps = [], 0, 0
    for _ in range(3):
        cx.barrier()
        t0 = time.perf_counter()
        s = post.sample((10_000 // cx.world,), x=x_o)
        cx.barrier()
        times.append(time.perf_counter() - t0)
        evals, steps = post._posterior_sampler.num_potential_evals, post._posterior_sampler.num_lock_steps
    sec = cx.max_over_ranks(sum(times) / len(times))
    if cx.rank == 0:
        print(json.dumps(_line(
            cx, "slice-sampling potential evals/sec (NLE nsf potential, 1000 chains)", cx.world * evals / sec, "evals/s",
            sec * 1e3, 3, 1,
            {"workload": "two-moons NLE likelihood_nn('nsf') 50k sims; slice_np_vectorized 1000 chains, 200 warm-up, "
                         "10k samples (BASELINE configs[2])", "parallelism": f"chains sharded over {cx.world} ranks",
             "api": "sbi_b200.posteriors.MCMCPosterior.sample"},
            {"scaling": "strong", "samples_per_s": 10_000 / sec, "lock_steps": steps,
             "us_per_lock_step": 1e6 * sec / max(steps, 1),
             "nle_training": {"samples_per_s": 45_000 * len(dur) / sum(dur), "epochs": len(dur)},
             "finite": bool(torch.isfinite(s).all()), "clocks": clocks.stop(), "gpu_launches": 2 * steps})))
    cx.finish()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="cfg2", choices=["cfg2", "cfg3", "cfg4", "cfg5"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-trainer", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's outputs as DIR/<name>.npy (cfg2)")
    args = ap.parse_args()
    if args.dump_outputs and (args.impl != "b200" or args.workload != "cfg2"):
        ap.error("--dump-outputs is implemented for the default workload (cfg2) of --impl b200")
    if args.impl == "reference":
        run_reference(args)
    else:
        {"cfg2": run_cfg2, "cfg3": run_cfg3, "cfg4": run_cfg4, "cfg5": run_cfg5}[args.workload](args)


if __name__ == "__main__":
    main()
