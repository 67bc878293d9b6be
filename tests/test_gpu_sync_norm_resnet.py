"""Converted ResNets (nn.SyncBatchNorm.convert_sync_batchnorm) on the sync batch-norm path, end to end.

W = 2 loopback replicas of resnet18 and resnet50, each after fuse_resnet and sync_batch_norm, train three SGD steps
under bf16 autocast with the gradients' mean over the ranks.  The reference is the same training with torch's own
nn.SyncBatchNorm, run by two threads over torch's multi-threaded process group (at W = 2 its sums are order-free):
every rank's loss at every step, and its parameters, running statistics and num_batches_tracked at the end, must
have the reference's bits.  One step must make no host synchronisation, and one step's trace must show no NCCL
kernel and no torch batch-norm kernel.  At world size 1 a converted resnet50 through prepare_model runs the local
fused sites (k_bn_stats<4>) and matches the unconverted model's fused step bit for bit."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm, train
from gpu_common import same_bits

torchvision = pytest.importorskip("torchvision")

pytestmark = pytest.mark.gpu

CL = torch.channels_last


@pytest.fixture(scope="module", autouse=True)
def deterministic_cudnn():
    saved = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = saved


def converted(name, seed):
    torch.manual_seed(seed)
    model = getattr(torchvision.models, name)(num_classes=10)
    model = nn.SyncBatchNorm.convert_sync_batchnorm(model)
    return model.cuda().to(memory_format=CL)


def batch(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, 3, 64, 64, device="cuda", generator=g).contiguous(memory_format=CL)
    return x, torch.randint(0, 10, (n,), device="cuda", generator=g)


def step(model, x, y):
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = F.cross_entropy(model(x), y)
    loss.backward()
    return loss.detach()


STEPS, SIZES = 3, [5, 3]   # an uneven split of a global batch of 8 over W = 2 ranks


def mean_grads(models):
    # the gradients' mean over the ranks: a sum of two (order-free), then 1/2, as both runs below compute it
    for ps in zip(*[m.parameters() for m in models]):
        mean = torch.sum(torch.stack([p.grad for p in ps]), dim=0).mul_(0.5)
        for p in ps:
            p.grad = mean.clone()


def reference_training(name):
    """torch's own nn.SyncBatchNorm, driven over torch's multi-threaded process group: one thread and one replica per
    rank.  Returns the losses of every step and the replicas."""
    import threading

    import torch.distributed as dist
    from torch.testing._internal.distributed.multi_threaded_pg import (ProcessLocalGroup, _install_threaded_pg,
                                                                       _uninstall_threaded_pg)

    W = len(SIZES)
    reps = [converted(name, 0) for _ in range(W)]
    losses = [[None] * STEPS for _ in range(W)]
    errors = []
    store = dist.HashStore()

    def all_gather_into_tensor(output, input, group=None, async_op=False):
        # The threaded group's all_gather_into_tensor cannot fill SyncBatchNorm's (1, W * n) output; gather a list
        # instead (SyncBatchNorm's own branch for gloo) and stack it in rank order.  Only the transport changes.
        parts = [torch.empty_like(input) for _ in range(W)]
        dist.all_gather(parts, input, group=group)
        output.view(W, -1).copy_(torch.stack(parts))

    # as torch's multi-threaded tests set up: each thread's process groups in its own registry and world
    torch._C._distributed_c10d._set_thread_isolation_mode(True)
    _install_threaded_pg()
    saved_gather, dist.all_gather_into_tensor = dist.all_gather_into_tensor, all_gather_into_tensor
    try:
        def worker(r):
            # each thread runs its own backward (autograd's shared device thread would serialise the two ranks'
            # backwards, and the first would wait forever in its all-reduce)
            torch.autograd.set_multithreading_enabled(False)
            try:
                dist.init_process_group("threaded", rank=r, world_size=W, store=store)
                opt = torch.optim.SGD(reps[r].parameters(), lr=0.05, momentum=0.9)
                for it in range(STEPS):
                    opt.zero_grad(set_to_none=True)
                    losses[r][it] = step(reps[r], *batch(SIZES[r], 100 * it + r))
                    for p in reps[r].parameters():
                        dist.all_reduce(p.grad)   # torch.sum over the stacked ranks
                        p.grad.mul_(0.5)
                    opt.step()
                torch.cuda.synchronize()
            except BaseException as e:  # noqa: BLE001
                errors.append(e)
                ProcessLocalGroup.exception_handle(e)   # wakes a peer waiting in a collective

        threads = [threading.Thread(target=worker, args=(r,)) for r in range(W)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        dist.all_gather_into_tensor = saved_gather
        _uninstall_threaded_pg()
        torch._C._distributed_c10d._set_thread_isolation_mode(False)
    if errors:
        raise errors[0]
    ProcessLocalGroup.reset()
    return losses, reps


@pytest.mark.parametrize("name", ["resnet18", "resnet50"])
def test_loopback_replicas_match_torch_sync_batch_norm(name):
    from ant_ray_b200.loopback import LoopbackWorld

    W = len(SIZES)
    want_losses, want = reference_training(name)
    base = fused_norm.fuse_resnet(converted(name, 0))
    # load every torch kernel of the step outside the world: with lazy module loading a first launch can wait for
    # the running kernels, which in a loopback world include a peer's collective (see test_gpu_sync_norm)
    warm = copy.deepcopy(base)
    for n in SIZES:   # cuDNN picks its kernels per shape
        step(warm, *batch(n, 0))
    torch.zeros(16, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    world = LoopbackWorld(W, device=0, key=f"syncbn-{name}", staging_bytes=1 << 20, max_blocks=8, timeout_ms=60000)
    try:
        reps = [fused_norm.sync_batch_norm(copy.deepcopy(base), world.comms[r]) for r in range(W)]
        opts = [torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9) for m in reps]
        for it in range(STEPS):
            data = [batch(SIZES[r], 100 * it + r) for r in range(W)]
            losses = [None] * W
            for o in opts:
                o.zero_grad(set_to_none=True)
            profile = it == 2
            if it == 1:
                torch.cuda.set_sync_debug_mode("error")
            try:
                if profile:
                    prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
                    prof.__enter__()
                world.run(lambda r, comm: losses.__setitem__(r, step(reps[r], *data[r])))
                if profile:
                    torch.cuda.synchronize()
                    prof.__exit__(None, None, None)
            finally:
                torch.cuda.set_sync_debug_mode("default")
            torch.cuda.synchronize()
            world.check()
            for r in range(W):
                assert same_bits(losses[r], want_losses[r][it]), f"step {it} rank {r}: loss differs from torch"
            mean_grads(reps)
            for o in opts:
                o.step()
        for r in range(W):
            got_sd, want_sd = reps[r].state_dict(), want[r].state_dict()
            assert list(got_sd) == list(want_sd)
            bad = [k for k in want_sd if not same_bits(got_sd[k], want_sd[k])]
            assert not bad, f"rank {r}: parameters / buffers differ from torch's SyncBatchNorm training: {bad[:8]}"
        names = [e.name for e in prof.events()]
        assert any("k_bn_sync_merge" in n for n in names)
        assert not [n for n in names if "nccl" in n.lower() or "batch_norm" in n], "NCCL or torch batch-norm kernels"
        nbt = [m.num_batches_tracked for m in reps[0].modules() if isinstance(m, nn.SyncBatchNorm)]
        assert all(int(t) == STEPS for t in nbt)
    finally:
        torch.cuda.synchronize()
        world.destroy()


def test_world_size_one_runs_the_local_fused_sites():
    plain = torchvision.models.resnet50(num_classes=10)
    plain = plain.cuda().to(memory_format=CL)
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    plain = train.prepare_model(plain)
    conv = train.prepare_model(conv)
    assert not hasattr(conv, "b200_norm_comm")
    x, y = batch(8, 1)
    want = step(plain, x, y)
    before = N.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        got = step(conv, x, y)
        torch.cuda.synchronize()
    assert N.launch_count() - before == 4 * 49   # the downsample branches stay on torch
    assert any("k_bn_stats<4>" in e.name for e in prof.events())
    assert same_bits(got, want)
    for (k, a), (_, b) in zip(conv.state_dict().items(), plain.state_dict().items()):
        assert same_bits(a, b), k
    for (k, a), (_, b) in zip(conv.named_parameters(), plain.named_parameters()):
        assert same_bits(a.grad, b.grad), k
