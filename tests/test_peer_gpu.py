"""Gradient sum over NVLink peer memory (csrc/peer.cu, parallel.PeerGradientSum) against NCCL
all-reduce, on two GPUs of one node (skipped on a single-GPU box)."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    import torch.distributed as dist
    from sbi_b200 import parallel
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    dev = torch.device("cuda", rank)
    P = 98025
    g = torch.Generator(device=dev).manual_seed(100 + rank)
    mask = (torch.rand(P, device=dev, generator=torch.Generator(device=dev).manual_seed(7)) > 0.1).to(torch.uint8)
    ex = parallel.PeerGradientSum(P)
    out = torch.zeros(P, device=dev)
    sumsq = torch.zeros(ex.n_sumsq, device=dev)
    step = torch.zeros(2, dtype=torch.int32, device=dev)
    loc = torch.zeros(P, device=dev)
    ok = True
    msgs = []

    def check(tag):
        nonlocal ok
        ref = loc.clone()
        dist.all_reduce(ref)
        torch.cuda.synchronize()
        if not torch.allclose(out, ref, rtol=1e-6, atol=1e-6):
            ok = False
            msgs.append(f"{tag}: sum mismatch {(out - ref).abs().max().item():.3e}")
        want = (out.double() * mask.double()).pow(2).sum().item()
        got = sumsq.double().sum().item()
        if abs(got - want) > 1e-5 * max(want, 1.0):
            ok = False
            msgs.append(f"{tag}: sumsq {got} vs {want}")
        both = [torch.zeros_like(out) for _ in range(world)]
        dist.all_gather(both, out)
        if not all(torch.equal(both[0], b) for b in both):
            ok = False
            msgs.append(f"{tag}: ranks differ bitwise")

    # eager steps
    for s in range(6):
        loc.copy_(torch.randn(P, device=dev, generator=g))
        ex.sum(loc, out, mask, sumsq, step)
        check(f"eager{s}")
        step[0] += 1
    # rewound step counter (warm-up then restore): stale flags must not satisfy the wait
    step[0] = 0
    for s in range(3):
        loc.copy_(torch.randn(P, device=dev, generator=g))
        ex.sum(loc, out, mask, sumsq, step)
        check(f"rewound{s}")
        step[0] += 1
    # CUDA graph replay
    torch.cuda.synchronize()
    dist.barrier()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ex.sum(loc, out, mask, sumsq, step)
        step[0] += 1
    torch.cuda.current_stream().wait_stream(side)
    check("pre-capture")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ex.sum(loc, out, mask, sumsq, step)
        step[0:1].add_(1)
    for s in range(4):
        loc.copy_(torch.randn(P, device=dev, generator=g))
        graph.replay()
        check(f"graph{s}")
    if ex.error():
        ok = False
        msgs.append("peer wait timed out")
    ex.close()
    q.put((rank, ok, msgs))
    dist.barrier()
    dist.destroy_process_group()


def test_peer_gradient_sum_matches_nccl(cuda_lib):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs on one node")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=240) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, ok, msgs in res:
        assert ok, (rank, msgs)


def _train_worker(rank, world, port, q):
    import math
    import torch.distributed as dist
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import NPE
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    D = 3
    torch.manual_seed(10 + rank)                       # every rank simulates its own shard
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((4000,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    torch.manual_seed(0)                               # same split / permutation stream on every rank
    inf = NPE(prior, density_estimator="nsf", device=f"cuda:{rank}").data_parallel("local")
    est = inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=6)
    flat = est.flat.data.clone()
    both = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(both, flat)
    same = all(torch.equal(both[0], b) for b in both)
    vl = inf.summary["validation_loss"]
    q.put((rank, same, [float(v) for v in vl]))
    dist.barrier()
    dist.destroy_process_group()


def test_data_parallel_training_two_gpus(cuda_lib):
    """NPE.data_parallel().train() on two GPUs: peer-memory gradient sum inside the per-epoch CUDA
    graph; the replicas end bit-identical and the validation loss goes down."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs on one node")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_train_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, same, vl in res:
        assert same, f"rank {rank}: replicas diverged"
        assert all(v == v for v in vl) and vl[-1] < vl[0], vl


def _run2(target, timeout=600, world=2, gpus=2):
    if torch.cuda.device_count() < gpus:
        pytest.skip(f"needs {gpus} GPUs on one node")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=timeout) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return sorted(res)


def _init(rank, world, port, backend="nccl"):
    """backend="gloo": every rank on cuda:0, gradients all-reduced through gloo (the NCCL-path code)."""
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    if backend == "nccl":
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    else:
        os.environ["SBI_B200_NCCL"] = "1"
        dist.init_process_group("gloo", rank=rank, world_size=world)
    return dist


def _lg(n, D, seed):
    import math
    from torch.distributions import MultivariateNormal
    torch.manual_seed(seed)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((n,))
    return prior, theta, theta + math.sqrt(0.1) * torch.randn_like(theta)


def _identical(dist, flat, world):
    if dist.get_backend() != "nccl":
        flat = flat.cpu()
    both = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(both, flat)
    return all(torch.equal(both[0], b) for b in both)


def _few_steps_worker(rank, world, port, q):
    """ADVICE r1: epochs of 1, 2 and 3 steps.  The warm-up epoch runs through the exchange and the
    optimizer state is rewound afterwards; the exchange's flags must not match the first real steps.
    At world size 2 the rank-order sum a+b equals NCCL's, so the peer path must reproduce the NCCL
    path up to the rounding of the clip norm."""
    from sbi_b200.inference import NPE
    dist = _init(rank, world, port)
    out = []
    for B in (3600, 1800, 1200):
        flats = []
        for nccl in ("0", "1"):
            os.environ["SBI_B200_NCCL"] = nccl
            prior, theta, x = _lg(4000, 3, 10 + rank)
            torch.manual_seed(0)
            inf = NPE(prior, density_estimator="nsf", device=f"cuda:{rank}").data_parallel("local")
            est = inf.append_simulations(theta, x).train(training_batch_size=B, max_num_epochs=4)
            flats.append(est.flat.data.clone())
        os.environ["SBI_B200_NCCL"] = "0"
        d = (flats[0] - flats[1]).abs()
        out.append((B, _identical(dist, flats[0], world), float((d > 5e-5).float().mean()), float(d.max())))
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def test_peer_exchange_epochs_of_one_to_three_steps(cuda_lib):
    for rank, out in _run2(_few_steps_worker):
        for B, same, frac_off, dmax in out:
            assert same, f"rank {rank} B={B}: replicas diverged"
            # (the two paths take the clip norm in different summation orders, so equality is up to
            # rounding; one stale gradient moves every weight by ~lr = 5e-4)
            assert frac_off < 1e-3, f"rank {rank} B={B}: peer path differs from the NCCL path " \
                                    f"({100 * frac_off:.2f}% of the weights by > 5e-5, max {dmax:.3e})"


def _global_worker(rank, world, port, q, backend="nccl"):
    """partition='global' (SURVEY 8e): same data on every rank, rank 0's split and epoch orders, rank r
    takes rows [r*B/G, (r+1)*B/G) of each global batch: the run equals the single-GPU run up to the
    summation order of the gradient partials."""
    from sbi_b200.inference import FMPE, NPE, NRE_B
    dist = _init(rank, world, port, backend)
    dev = f"cuda:{rank}" if backend == "nccl" else "cuda:0"
    prior, theta, x = _lg(4000, 3, 5)                   # identical data on every rank
    res = {}
    torch.manual_seed(0)
    inf = NPE(prior, density_estimator="nsf", device=dev).data_parallel("global")
    est = inf.append_simulations(theta, x).train(training_batch_size=400, max_num_epochs=3)
    res["npe_same"] = _identical(dist, est.flat.data, world)
    res["npe_val"] = list(inf.summary["validation_loss"])
    res["npe_train"] = list(inf.summary["training_loss"])
    if rank == 0:   # the single-process run on the same seeds
        torch.manual_seed(0)
        solo = NPE(prior, density_estimator="nsf", device="cuda:0")
        solo.append_simulations(theta, x).train(training_batch_size=400, max_num_epochs=3)
        res["solo_val"] = list(solo.summary["validation_loss"])
        res["solo_train"] = list(solo.summary["training_loss"])
    dist.barrier()
    torch.manual_seed(1)
    fm = FMPE(prior, device=dev).data_parallel("global")
    e2 = fm.append_simulations(theta, x).train(training_batch_size=400, max_num_epochs=4)
    res["fm_same"] = _identical(dist, e2.flat.data, world)
    res["fm_train"] = list(fm.summary["training_loss"])
    torch.manual_seed(2)
    nre = NRE_B(prior, device=dev).data_parallel("global")
    e3 = nre.append_simulations(theta, x).train(training_batch_size=400, max_num_epochs=4)
    res["nre_same"] = _identical(dist, e3.flat.data, world)
    res["nre_val"] = list(nre.summary["validation_loss"])
    torch.manual_seed(3 + rank)                         # weak mode for the other two trainers
    fm = FMPE(prior, device=dev).data_parallel("local")
    e4 = fm.append_simulations(theta, x).train(training_batch_size=400, max_num_epochs=3)
    res["fm_local_same"] = _identical(dist, e4.flat.data, world)
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()


def _check_global(out):
    for rank, res in out.items():
        for k in ("npe_same", "fm_same", "nre_same", "fm_local_same"):
            assert res[k], f"rank {rank}: {k} failed (replicas diverged)"
        assert res["fm_train"][-1] < res["fm_train"][0]
        assert res["nre_val"][-1] < res["nre_val"][0]
    r0 = out[0]
    # same batches, same updates: the loss curves of the 2-GPU and the 1-GPU run agree
    for a, b in zip(r0["npe_train"] + r0["npe_val"], r0["solo_train"] + r0["solo_val"]):
        assert abs(a - b) < 2e-3 * max(1.0, abs(b)), (r0["npe_train"], r0["solo_train"], r0["npe_val"], r0["solo_val"])


def test_global_batch_data_parallel_all_trainers(cuda_lib):
    _check_global(dict(_run2(_global_worker, timeout=900)))


def test_global_batch_data_parallel_all_reduce_one_gpu(cuda_lib):
    """The same runs as two gloo processes sharing cuda:0 with SBI_B200_NCCL=1: every trainer's all-reduce
    path (eager launches, no peer memory)."""
    import functools
    _check_global(dict(_run2(functools.partial(_global_worker, backend="gloo"), timeout=900, gpus=1)))
