"""Fused batch norm for the training step and eval forward of ResNets, DenseNets, Inception v3, GoogLeNet, ShuffleNetV2,
VGG-BN and torchvision's Conv2dNormActivation blocks (libb200coll.so, norm_kernels.cuh, norm_infer.cuh, norm_act.cuh,
norm_res.cuh, norm_cat.cuh, norm_slice.cuh, norm_shuffle.cuh, norm_pool2.cuh), and the
squeeze-and-excitation of EfficientNet and MobileNetV3 blocks (se_kernels.cuh).

Every batch norm of a torchvision ResNet is followed by a ReLU, by `+= identity` and a ReLU (a block's tail), or
by nothing (a downsample branch).  In bf16 training torch runs the first two kinds as separate memory-bound
passes: batch norm, ReLU and the residual add forward; threshold_backward and batch norm backward.
`fuse_resnet` swaps a model's torchvision `ResNet`, `Bottleneck` and `BasicBlock` classes for subclasses whose
forward runs each such site as one native call per direction, which writes its output once and folds the ReLU
mask into the backward.  A downsample branch's batch norm runs inside its block tail's call (`bn_add_relu_downsample`),
and the stem's batch norm, ReLU and max-pool are one call (`bn_relu_maxpool`).  The kernels reproduce torch's own channels-last kernels, reduction order included, so
outputs, gradients and running statistics are bit-identical to eager torch.

A site runs fused when it is in training mode, its input is a bf16 channels-last CUDA tensor with more than one
value per channel, a channel stride of 1 and at most 131072 channels, its batch norm is
a plain `BatchNorm2d` with fp32 affine weight and bias, tracked running statistics and a numeric momentum,
torch would run it on its native kernels (`torch._C._select_batch_norm_backend`), and the hook rule holds.
Otherwise the block runs the parent class's ops, so the choice never changes a result.

The hook rule, the same at every site of every kind below, training and eval, local and sync: the kernels replace
the calls of the batch norm and of other modules (the ReLU or activation, the stem's max-pool, a downsample branch's
Sequential and batch norm, an inverted-residual block's projection and stochastic depth, the squeeze-excitation's
average pool), so a site runs on them only where none of those modules has a forward, forward-pre, backward or
backward-pre hook and no global module hook is registered.  Otherwise the modules are called and every hook runs as
in eager torch.  `_site` decides every batch-norm site: the hook rule, the other operands, then an eval site, a sync
site or a local site.  The stem's max-pool and a downsample branch are checked for their own hooks with their shape
and structure (`_pool_fusable`, `_downsample_bn`), before the site asks `_site`.

Eval mode: where no gradient is recorded (`torch.no_grad()`, `torch.inference_mode()`, or nothing the site reads
requires grad), the same four kinds of site run as one native launch each on the eval kernels, which read the
running statistics and write only the site's output (no running statistic, no `num_batches_tracked`), with the bits
of eager torch's eval batch norm and the ReLU, add and max-pool after it.  A site runs there when its batch norm is
a `BatchNorm2d`, or a SyncBatchNorm (which torch does not synchronise in eval), in eval mode with running
statistics and a positive eps; its weight, bias and running statistics are contiguous on the input's device and
all fp32 or all bf16 (a model cast to bf16); the input is a non-empty bf16 channels-last CUDA tensor with a channel
stride of 1 and fewer than 2^31 elements; torch would run it on its native kernels; and the hook rule holds.
Otherwise the site runs torch's ops.  With gradients recorded,
eval runs the parent classes' forward.

Conv2dNormActivation: `fuse_model` also swaps every torchvision `Conv2dNormActivation` that ends in an nn.ReLU6,
nn.SiLU or nn.Hardswish (MobileNetV2 / V3, EfficientNet) for `FusedConv2dNormActivation`, whose batch norm and
activation run as one site per direction (`bn_act`, norm_act.cuh): the forward writes act(bn(x)) with eager torch's
bits, and the backward recomputes bn(x) from x instead of saving it.  `bn_act` runs nn.ReLU on the ReLU sites above.  The
conditions are those above, the hook rule covering the activation; in eval without autograd recording the site is
one launch.  A sync site with one of those activations runs the sync batch norm alone, then the activation.

Inverted-residual blocks: `fuse_model` also swaps torchvision's MobileNetV2 / V3 `InvertedResidual` and
EfficientNet's `MBConv` for subclasses whose projection batch norm (the 1x1 convolution's, without activation) runs
with what follows it as one site per direction (`bn_res`, norm_res.cuh): nothing, the residual add, or EfficientNet's
stochastic depth ("row" mode, its noise built by torchvision's own torch calls) and the add.  The conditions are those
above, the hook rule covering the block's Sequential, the projection and the stochastic depth; in eval without
autograd recording the site is one launch.

Squeeze-and-excitation: inside those swapped MBConv and MobileNetV3 blocks, `fuse_model` also swaps torchvision's
`SqueezeExcitation` for `FusedSqueezeExcitation`, whose average pool and scale `s * x` run on native kernels (the
squeeze path, fc1, activation, fc2 and scale activation, still runs as modules on torch): in training, a pool and a
scale forward, and backward one reduce (s's gradient, the sum over H, W of dy * x) and one elementwise kernel that
writes x's whole gradient (dy * s plus the mean's gp / HW) once; without autograd recording, the two forward launches.
The two sums keep the launch shape and order of torch's reduce kernel, so outputs and gradients are eager torch's bits.
A site runs there when x is a non-empty bf16 channels-last CUDA tensor with a channel stride of 1, fewer than 2^30
elements and not one channel over several rows, the module's avgpool is exactly an nn.AdaptiveAvgPool2d(1), and the
hook rule holds for it; otherwise the parent's forward runs.  A squeeze path that returns
anything but a bf16 [N, C, 1, 1] on x's device gets torch's `s * x`, and a gradient that arrives in another layout
than channels-last torch's backward ops.

DenseNet: `fuse_model` also swaps torchvision's `_DenseLayer`, `_DenseBlock` and `DenseNet` for subclasses whose
`relu(bn(torch.cat(features, 1)))` sites (each dense layer's norm1 / relu1, each transition's norm / relu, and norm5
with DenseNet's functional ReLU) run as concatenation sites (`bn_relu_cat`, norm_cat.cuh) that read the earlier feature
maps where they lie: no concatenation is written or saved, and each feature map's gradient is its channels of the
one dx the backward writes, as torch's CatBackward hands them out.  The site runs where every segment is a bf16
channels-last CUDA tensor with a channel stride of 1, a multiple of 8 channels and a data pointer on the 16-byte grid,
alike in N, H, W and device, at most 64 of them, and the batch norm, decided on a tensor of the concatenation's shape
and layout, is an eval or a local site by the rules above; anything else, a sync site included, runs torch.cat and
bn_relu.  Each norm2 / relu2 is a bn_relu site and the stem a bn_relu_maxpool site.

Inception v3 and GoogLeNet: `fuse_model` also swaps torchvision's `BasicConv2d` (of both models), whose
`F.relu(bn(conv(x)), inplace=True)` then runs as a bn_relu eval or local site (a sync batch norm keeps the module's
forward), and the Inception modules (`InceptionA` to `InceptionE`, GoogLeNet's `Inception`), whose `torch.cat` of their
branches is built in place: each branch's last batch norm and ReLU is a slice site (`bn_relu_concat`, norm_slice.cuh)
that writes its output straight into its channels of the module's channels-last output, and a max-pool branch is
copied there as torch.cat copies it; InceptionE's inner concatenations flatten into the outer one.  No branch output is
written or kept for the backward, whose gradient reads each site's channels of dy in place, and every result is eager
torch's bits.  A module runs there when every branch operand is a bf16 channels-last CUDA tensor with a multiple of 8
channels on the 16-byte grid and every site is an eval or a local site by the rules above; where a branch-ending
BasicConv2d, its batch norm or a GoogLeNet branch Sequential has a hook, a global hook is registered, or in eval with
gradients recorded, the module runs its parent's forward, and where only the operands or the sites fail, it runs the
batch norms and ReLUs as modules and torch.cat.  The convolutions run in torchvision's order before any branch's last
batch norm, so the backward adds the module input's branch gradients in eager torch's order.

ShuffleNetV2: `fuse_model` also swaps torchvision's ShuffleNetV2 `InvertedResidual` and `ShuffleNetV2`.  A block walks
its branches module by module: branch2's first batch norm and ReLU is a bn_relu site, each batch norm after a depthwise
convolution a bn_res site without identity, and the block's end, `channel_shuffle(torch.cat((x1 or branch1(x),
branch2(x2)), 1), 2)`, is one block-end site (`bn_relu_shuffle`, norm_shuffle.cuh) over the branches' last batch norms
and ReLUs that writes the shuffled, contiguous NCHW output directly: no branch output or concatenation is written, and
the backward reads the output's gradient in place and gives x1 the gradient eager torch's view / transpose / reshape
chain gives it.  The model's stem is a bn_relu_maxpool site and conv5 a bn_relu site.  Any branch width runs there (58
and 116 are not multiples of 8).  A block runs there when its branch operands are bf16 channels-last CUDA tensors of
one shape with at most 65536 channels, a stride-1 block's input is contiguous NCHW, and every site is an eval or a
local site by the rules above; where a branch Sequential, a tail batch norm or its ReLU has a hook, a global hook is
registered, or in eval with gradients recorded, the block runs its parent's forward, and where only the operands or the
sites fail, the modules, torch.cat and channel_shuffle.  Block ends are never sync sites.

VGG-BN: `fuse_model` also swaps torchvision's `VGG`, whose forward walks `features` group by group.  Each stage's end,
Conv2d, batch norm, ReLU and nn.MaxPool2d(2, 2), is one stage-end site (`bn_relu_maxpool`, norm_pool2.cuh) that writes
only the pooled output and one argmax byte per pooled element, which also stands in for the ReLU's mask; relu(bn(x)) is
never written or saved, and the backward rebuilds the batch norm's output gradient from the pooled gradient and those
bytes.  Every other Conv2d, batch norm and ReLU is a bn_relu site, and any other module runs as a module, so a VGG
without batch norm computes torchvision's ops.  A stage end runs there when the max-pool is exactly nn.MaxPool2d(2, 2)
(padding 0, dilation 1, floor mode, no indices) without a hook, the input has at least 2 rows and 2 columns (torch
raises below that), and the batch norm is an eval or a local site by the rules above; a sync batch norm there runs its
own module forward, as at the stem.  Where `features` is not an nn.Sequential or has a hook, a global hook is
registered, or in eval with gradients recorded, the model runs its parent's forward; a hook on a batch norm, ReLU or
max-pool makes that group call its modules.

Sync batch norm: `sync_batch_norm(model, comm)` gives every `nn.SyncBatchNorm` of the world group the subclass
`FusedSyncBatchNorm`, which records a peer-memory communicator.  Where such a module runs with a communicator of
more than one rank (a "sync site"), its statistics are gathered and its gradient sums reduced over that
communicator instead of torch's NCCL process group, with one native call per direction that also fuses the ReLU and
the residual add at ResNet positions; the results have the bits of torch's SyncBatchNorm function (ranks folded in
rank order).  Whether a site syncs depends only on the module and the input's layout, never on the rank's batch
size, so every rank joins the same collectives: a rank with an empty batch still contributes its zero row.  Where
the hook rule fails, the block calls the FusedSyncBatchNorm, whose own forward is the sync site without ReLU.  A
SyncBatchNorm that torch would not synchronise (no process group, or one rank) runs the local fused site above,
which is what torch's F.batch_norm computes.
"""
import ctypes
import numbers

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from . import _native as N

_lib = None
# (device index, stream) -> (bytes, pointer, zero-initialised uint8 tensor).  One buffer per stream serves every
# channel count (the library keeps its semaphores in a region no call's staging overlaps); calls on one stream
# are ordered.
_scratch = {}
_scratch_need = {}   # (channels, world or None) -> the library's scratch bytes; 0: more channels than the kernels take
# the squeeze-excitation sites' scratch, as _scratch (its semaphores sit at the start as well, so it is a buffer of its own)
_se_scratch = {}
_se_need = {}        # (device index, n, c, hw) -> b200c_se_scratch_bytes
_NATIVE = torch._C._BatchNormBackend.Native
# the current stream's handle without building a torch.cuda.Stream object: each step makes 98 fused calls
_raw_stream = torch._C._cuda_getCurrentRawStream


def _native_lib():
    global _lib
    if _lib is None:
        _lib = N.load()
    return _lib


def _scratch_bytes(channels, world=None):
    """The scratch a site of `channels` needs: a local site's, with `world` a sync site's over that many ranks, or with
    world "dual" a dual tail's (a tail and its downsample branch's batch norm)."""
    key = (channels, world)
    need = _scratch_need.get(key)
    if need is None:
        lib = _native_lib()
        if world == "dual":
            need = lib.b200c_bn_dual_scratch_bytes(channels)
        else:
            need = lib.b200c_bn_scratch_bytes(channels) if world is None else lib.b200c_bn_sync_scratch_bytes(channels, world)
        need = _scratch_need[key] = int(need)
    return need


def _scratch_ptr(device, stream, need, table=_scratch):
    key = (device.index, stream)
    entry = table.get(key)
    if entry is None or entry[0] < need:
        buf = torch.zeros(need, dtype=torch.uint8, device=device)
        entry = table[key] = (need, buf.data_ptr(), buf)
    return entry[1]


def _stream_scratch(x, comm=None, dual=False):
    """The stream a training site's calls run on and its scratch there: the current stream and a local site's scratch
    for x's channels (with `dual` a dual tail's), or with `comm` the communicator's stream and a sync site's scratch."""
    if comm is not None:
        stream = comm.stream().cuda_stream
        return stream, _scratch_ptr(x.device, stream, _scratch_bytes(x.shape[1], comm.world_size))
    stream = _raw_stream(x.device.index)
    return stream, _scratch_ptr(x.device, stream, _scratch_bytes(x.shape[1], "dual" if dual else None))


def _forward_args(x, bn, weight, bias, comm=None, dual=False):
    """What every training site's forward call takes for its batch norm `bn`: the stats tensor it writes, [save_mean (C)
    | save_invstd (C)] (followed at a sync site by norm_fct, the backward's 1 / rows of all ranks, whose statistics are
    the global ones), the seven pointers weight, bias, running_mean, running_var, num_batches_tracked or None,
    save_mean and save_invstd, and _stream_scratch's stream and scratch."""
    c = x.shape[1]
    stats = torch.empty(2 * c + (comm is not None), dtype=torch.float32, device=x.device)
    mean = stats.data_ptr()
    nbt = bn.num_batches_tracked
    params = (weight.data_ptr(), bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
              nbt.data_ptr() if nbt is not None else None, mean, mean + 4 * c)
    return (stats, params, *_stream_scratch(x, comm, dual))


def _backward_args(x, comm=None, dual=False):
    """What every training site's backward call writes for its batch norm of input x, dx, grad_weight and grad_bias,
    and _stream_scratch's stream and scratch."""
    c = x.shape[1]
    return (torch.empty_like(x), torch.empty(c, dtype=torch.float32, device=x.device),
            torch.empty(c, dtype=torch.float32, device=x.device), *_stream_scratch(x, comm, dual))


def _torch_backward(g, x, weight, stats, eps):
    """Eager torch's batch-norm backward (dx, grad_weight, grad_bias) of a training site for g, the gradient of its
    output: the sites whose gradient arrives in another layout than channels-last run it, as eager torch then runs its
    NCHW kernels, whose sums round differently.  The running statistics are not read in training mode."""
    c = x.shape[1]
    return torch.ops.aten.native_batch_norm_backward(g, x, weight, None, None, stats[:c], stats[c:], True, eps, [True, True, True])


def _pooled_like(x):
    """An empty channels-last output of the stem's nn.MaxPool2d(3, 2, 1) over x."""
    n, c, h, w = x.shape
    return torch.empty((n, c, (h - 1) // 2 + 1, (w - 1) // 2 + 1), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)


def _pooled2_like(x):
    """An empty channels-last output of VGG's nn.MaxPool2d(2, 2) over x: floor(h / 2) x floor(w / 2)."""
    n, c, h, w = x.shape
    return torch.empty((n, c, h // 2, w // 2), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)


class _FusedBatchNorm(torch.autograd.Function):
    """relu(bn(x)) or, with `identity`, relu(bn(x) + identity) in training mode.

    With `pair` the output is returned twice, as y and a view of it, for a block tail whose output feeds both
    branches of the next block: autograd then hands the backward the two branches' gradients apart (None for an
    unused one), and the kernel sums them as autograd would.  Where C % 8 == 0 the forward writes the ReLU's mask
    as bits and the backward reads those instead of y.

    With `comm` (a PeerMemoryComm) the site is a sync site over its ranks; `relu` False then runs bn(x) alone, the
    forward of a SyncBatchNorm with nothing fused after it."""

    @staticmethod
    def forward(ctx, x, identity, weight, bias, bn, pair, comm=None, relu=True):
        lib = _native_lib()
        c = x.shape[1]
        m = x.numel() // c
        y = torch.empty_like(x)
        id_ptr = identity.data_ptr() if identity is not None else None
        ctx.residual = identity is not None
        ctx.comm, ctx.relu = comm, relu
        ctx.set_materialize_grads(False)
        # what the backward reads of the ReLU: its mask (where C % 8 == 0), else y; nothing at a site without ReLU, whose
        # output may then be modified in place (an inplace ReLU or `+= identity` after a SyncBatchNorm)
        masked = relu and c % 8 == 0
        relu_src = torch.empty(m * c // 8, dtype=torch.uint8, device=x.device) if masked else y if relu else None
        mask_ptr = relu_src.data_ptr() if masked else None
        stats, params, stream, scratch = _forward_args(x, bn, weight, bias, comm)
        if comm is not None:
            N.check(lib.b200c_bn_sync_forward(comm._h(), x.data_ptr(), id_ptr, y.data_ptr(), mask_ptr, int(relu), *params,
                                              stats.data_ptr() + 8 * c, m, c, bn.momentum, bn.eps, scratch, stream))
        elif masked:
            N.check(lib.b200c_bn_forward_mask(x.data_ptr(), id_ptr, y.data_ptr(), mask_ptr, *params, m, c, bn.momentum, bn.eps,
                                              scratch, stream))
        else:
            N.check(lib.b200c_bn_forward(x.data_ptr(), id_ptr, y.data_ptr(), *params, m, c, bn.momentum, bn.eps, scratch, stream))
        ctx.save_for_backward(x, relu_src, weight, stats)
        return (y, y.view_as(y)) if pair else y

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        grads = [g.contiguous(memory_format=torch.channels_last) for g in grads if g is not None]
        x, relu_src, weight, stats = ctx.saved_tensors
        comm = ctx.comm
        if not grads:
            if comm is None:
                return None, None, None, None, None, None, None, None
            # the other ranks wait in this site's all-reduce: join it with a zero gradient
            grads = [torch.zeros_like(x, memory_format=torch.channels_last)]
        lib = _native_lib()
        c = x.shape[1]
        m = x.numel() // c
        dx, grad_weight, grad_bias, stream, scratch = _backward_args(x, comm)
        d_identity = torch.empty_like(x) if ctx.residual else None
        mean = stats.data_ptr()
        did_ptr = d_identity.data_ptr() if d_identity is not None else None
        # the forward's relu_src: the mask, y, or nothing
        mask = relu_src.data_ptr() if relu_src is not None and relu_src.dtype == torch.uint8 else None
        y = relu_src.data_ptr() if relu_src is not None and mask is None else None
        dy2 = grads[1].data_ptr() if len(grads) == 2 else None
        if comm is not None:
            N.check(lib.b200c_bn_sync_backward(comm._h(), grads[0].data_ptr(), dy2, y, mask, int(ctx.relu), x.data_ptr(),
                                               did_ptr, dx.data_ptr(), weight.data_ptr(), mean, mean + 4 * c, mean + 8 * c,
                                               grad_weight.data_ptr(), grad_bias.data_ptr(), m, c, scratch, stream))
            if m == 0:
                # as torch's SyncBatchNorm: no gradient for an empty input, nor for weight and bias from this rank
                return None, d_identity, None, None, None, None, None, None
            return dx, d_identity, grad_weight, grad_bias, None, None, None, None
        site = (x.data_ptr(), did_ptr, dx.data_ptr(), weight.data_ptr(), mean, mean + 4 * c, grad_weight.data_ptr(),
                grad_bias.data_ptr(), m, c, scratch, stream)
        if mask is not None:
            N.check(lib.b200c_bn_backward_mask(grads[0].data_ptr(), dy2, mask, *site))
        else:
            dy = grads[0] + grads[1] if dy2 is not None else grads[0]   # this call takes one gradient
            N.check(lib.b200c_bn_backward(dy.data_ptr(), y, *site))
        return dx, d_identity, grad_weight, grad_bias, None, None, None, None


class _FusedBatchNormDual(torch.autograd.Function):
    """relu(bn(x) + bn_ds(x_ds)) in training mode: a block tail whose identity is its downsample branch's batch norm.
    bn_ds(x_ds) is never written, and the backward writes dx and dx_ds from one walk over g.  `pair` as in
    _FusedBatchNorm."""

    @staticmethod
    def forward(ctx, x, x_ds, weight, bias, weight_ds, bias_ds, bn, bn_ds, pair):
        c = x.shape[1]
        m = x.numel() // c
        y = torch.empty_like(x)
        ctx.set_materialize_grads(False)
        masked = c % 8 == 0
        relu_src = torch.empty(m * c // 8, dtype=torch.uint8, device=x.device) if masked else y
        stats, params, stream, scratch = _forward_args(x, bn, weight, bias, dual=True)
        stats_ds, params_ds, _, _ = _forward_args(x_ds, bn_ds, weight_ds, bias_ds, dual=True)
        N.check(_native_lib().b200c_bn_forward_dual(x.data_ptr(), x_ds.data_ptr(), y.data_ptr(), relu_src.data_ptr() if masked else None,
                                                    *params, bn.momentum, bn.eps, *params_ds, bn_ds.momentum, bn_ds.eps, m, c,
                                                    scratch, stream))
        ctx.save_for_backward(x, x_ds, relu_src, weight, weight_ds, stats, stats_ds)
        return (y, y.view_as(y)) if pair else y

    @staticmethod
    @once_differentiable
    def backward(ctx, *grads):
        grads = [g.contiguous(memory_format=torch.channels_last) for g in grads if g is not None]
        if not grads:
            return (None,) * 9
        x, x_ds, relu_src, weight, weight_ds, stats, stats_ds = ctx.saved_tensors
        c = x.shape[1]
        dx, dw, db, stream, scratch = _backward_args(x, dual=True)
        dx_ds, dw_ds, db_ds, _, _ = _backward_args(x_ds, dual=True)
        mean, mean_ds = stats.data_ptr(), stats_ds.data_ptr()
        masked = relu_src.dtype == torch.uint8
        N.check(_native_lib().b200c_bn_backward_dual(
            grads[0].data_ptr(), grads[1].data_ptr() if len(grads) == 2 else None, None if masked else relu_src.data_ptr(),
            relu_src.data_ptr() if masked else None, x.data_ptr(), x_ds.data_ptr(), dx.data_ptr(), dx_ds.data_ptr(),
            weight.data_ptr(), mean, mean + 4 * c, dw.data_ptr(), db.data_ptr(), weight_ds.data_ptr(), mean_ds, mean_ds + 4 * c,
            dw_ds.data_ptr(), db_ds.data_ptr(), x.numel() // c, c, scratch, stream))
        return dx, dx_ds, dw, db, dw_ds, db_ds, None, None, None


class _FusedBatchNormPool(torch.autograd.Function):
    """maxpool(relu(bn(x))) in training mode, maxpool being nn.MaxPool2d(3, 2, 1): the ResNet stem.  The forward writes
    the pooled output and one argmax byte per pooled element, never relu(bn(x)) itself; the backward takes the pooled
    output's gradient."""

    @staticmethod
    def forward(ctx, x, weight, bias, bn):
        n, c, h, w = x.shape
        y = _pooled_like(x)
        argmax = torch.empty(y.numel(), dtype=torch.uint8, device=x.device)
        stats, params, stream, scratch = _forward_args(x, bn, weight, bias)
        N.check(_native_lib().b200c_bn_forward_pool(x.data_ptr(), y.data_ptr(), argmax.data_ptr(), *params, n, h, w, c,
                                                    bn.momentum, bn.eps, scratch, stream))
        ctx.save_for_backward(x, argmax, weight, stats)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        if dy is None:
            return None, None, None, None
        dy = dy.contiguous(memory_format=torch.channels_last)
        x, argmax, weight, stats = ctx.saved_tensors
        n, c, h, w = x.shape
        g = torch.empty_like(x)
        dx, grad_weight, grad_bias, stream, scratch = _backward_args(x)
        mean = stats.data_ptr()
        N.check(_native_lib().b200c_bn_backward_pool(dy.data_ptr(), argmax.data_ptr(), x.data_ptr(), g.data_ptr(), dx.data_ptr(),
                                                     weight.data_ptr(), mean, mean + 4 * c, grad_weight.data_ptr(),
                                                     grad_bias.data_ptr(), n, h, w, c, scratch, stream))
        return dx, grad_weight, grad_bias, None


class _FusedBatchNormPool2(torch.autograd.Function):
    """maxpool(relu(bn(x))) in training mode, maxpool being nn.MaxPool2d(2, 2): the end of a VGG stage.  The forward
    writes the pooled output and one argmax byte per pooled element, never relu(bn(x)) itself; the backward takes the
    pooled output's gradient and rebuilds the batch norm's output gradient from it and the argmax bytes."""

    @staticmethod
    def forward(ctx, x, weight, bias, bn):
        n, c, h, w = x.shape
        y = _pooled2_like(x)
        argmax = torch.empty(y.numel(), dtype=torch.uint8, device=x.device)
        stats, params, stream, scratch = _forward_args(x, bn, weight, bias)
        N.check(_native_lib().b200c_bn_forward_pool2(x.data_ptr(), y.data_ptr(), argmax.data_ptr(), *params, n, h, w, c,
                                                     bn.momentum, bn.eps, scratch, stream))
        ctx.save_for_backward(x, argmax, weight, stats)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        if dy is None:
            return None, None, None, None
        dy = dy.contiguous(memory_format=torch.channels_last)
        x, argmax, weight, stats = ctx.saved_tensors
        n, c, h, w = x.shape
        dx, grad_weight, grad_bias, stream, scratch = _backward_args(x)
        mean = stats.data_ptr()
        N.check(_native_lib().b200c_bn_backward_pool2(dy.data_ptr(), argmax.data_ptr(), x.data_ptr(), dx.data_ptr(), weight.data_ptr(),
                                                      mean, mean + 4 * c, grad_weight.data_ptr(), grad_bias.data_ptr(), n, h, w, c,
                                                      scratch, stream))
        return dx, grad_weight, grad_bias, None


# eager torch's backward of each activation, g of (dy, t)
_ACT_BACKWARD = {N.ACT_RELU6: lambda dy, t: torch.ops.aten.hardtanh_backward(dy, t, 0.0, 6.0),
                 N.ACT_SILU: torch.ops.aten.silu_backward, N.ACT_HARDSWISH: torch.ops.aten.hardswish_backward}


class _FusedBatchNormAct(torch.autograd.Function):
    """act(bn(x)) in training mode, act being ReLU6, SiLU or Hardswish (`code`, the library's b200c_act_t).  The
    batch norm's output is never written: the backward recomputes it from x, the saved statistics, weight and bias, and
    writes the activation's gradient g for the batch norm's elementwise backward.

    A gradient that arrives in another layout than channels-last (at the last block before a model's average pool)
    makes eager torch's activation backward write g in that layout, and its batch-norm backward then runs its NCHW
    kernels, whose sums round differently.  There the backward runs those torch ops on t recomputed by torch's own
    transform, so the bits stay eager torch's."""

    @staticmethod
    def forward(ctx, x, weight, bias, bn, code):
        c = x.shape[1]
        y = torch.empty_like(x)
        stats, params, stream, scratch = _forward_args(x, bn, weight, bias)
        N.check(_native_lib().b200c_bn_forward_act(x.data_ptr(), y.data_ptr(), *params, code, x.numel() // c, c, bn.momentum, bn.eps,
                                                   scratch, stream))
        ctx.code, ctx.eps = code, bn.eps
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(x, weight, bias, stats)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        if dy is None:
            return None, None, None, None, None
        x, weight, bias, stats = ctx.saved_tensors
        c = x.shape[1]
        if not dy.is_contiguous(memory_format=torch.channels_last):
            t = torch.batch_norm_elemt(x, weight, bias, stats[:c], stats[c:], ctx.eps)
            return (*_torch_backward(_ACT_BACKWARD[ctx.code](dy, t), x, weight, stats, ctx.eps), None, None)
        g = torch.empty_like(x)
        dx, grad_weight, grad_bias, stream, scratch = _backward_args(x)
        mean = stats.data_ptr()
        N.check(_native_lib().b200c_bn_backward_act(dy.data_ptr(), x.data_ptr(), g.data_ptr(), dx.data_ptr(), weight.data_ptr(),
                                                    bias.data_ptr(), mean, mean + 4 * c, grad_weight.data_ptr(), grad_bias.data_ptr(),
                                                    ctx.code, x.numel() // c, c, scratch, stream))
        return dx, grad_weight, grad_bias, None, None


class _FusedBatchNormRes(torch.autograd.Function):
    """bn(x), bn(x) + identity or, with `noise`, bf16(bn(x) * noise) + identity in training mode: the projection batch
    norm of an inverted-residual block, and the stochastic depth (`noise`, torchvision's [N, 1, 1, 1] bf16 "row" noise)
    and residual add after it.  Only the sum is written.  The identity's gradient is dy itself; with noise the backward
    writes stochastic depth's g = bf16(dy * noise) for the batch norm's elementwise backward.

    A gradient that arrives in another layout than channels-last makes eager torch's mul write g in that layout and its
    batch-norm backward run its NCHW kernels; there the backward runs those torch ops, as _FusedBatchNormAct does."""

    @staticmethod
    def forward(ctx, x, identity, weight, bias, bn, noise):
        c = x.shape[1]
        y = torch.empty_like(x)
        stats, params, stream, scratch = _forward_args(x, bn, weight, bias)
        N.check(_native_lib().b200c_bn_forward_res(x.data_ptr(), identity.data_ptr() if identity is not None else None,
                                                   noise.data_ptr() if noise is not None else None, x.shape[2] * x.shape[3],
                                                   y.data_ptr(), *params, x.numel() // c, c, bn.momentum, bn.eps, scratch, stream))
        ctx.residual, ctx.eps = identity is not None, bn.eps
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(x, weight, stats, noise)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        if dy is None:
            return None, None, None, None, None, None
        x, weight, stats, noise = ctx.saved_tensors
        c = x.shape[1]
        d_identity = dy if ctx.residual else None
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dx, grad_weight, grad_bias = _torch_backward(dy * noise if noise is not None else dy, x, weight, stats, ctx.eps)
            return dx, d_identity, grad_weight, grad_bias, None, None
        g = torch.empty_like(x) if noise is not None else None
        dx, grad_weight, grad_bias, stream, scratch = _backward_args(x)
        mean = stats.data_ptr()
        N.check(_native_lib().b200c_bn_backward_res(dy.data_ptr(), noise.data_ptr() if noise is not None else None,
                                                    x.shape[2] * x.shape[3], x.data_ptr(), g.data_ptr() if g is not None else None,
                                                    dx.data_ptr(), weight.data_ptr(), mean, mean + 4 * c, grad_weight.data_ptr(),
                                                    grad_bias.data_ptr(), x.numel() // c, c, scratch, stream))
        return dx, d_identity, grad_weight, grad_bias, None, None


def _activation(t):
    # With one channel, NCHW strides also pass the channels-last check, but torch runs its NCHW statistics kernel
    # unless stride(1) == 1 (batch_norm_choose_impl), so the channel stride must be 1 as well.
    return (t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last)
            and t.stride(1) == 1)


def _torch_syncs(bn):
    """Whether torch's SyncBatchNorm.forward would synchronise `bn` (its need_sync, in training mode)."""
    if not (dist.is_available() and dist.is_initialized()):
        return False
    return dist.get_world_size(bn.process_group or dist.group.WORLD) > 1


def _module_ok(bn):
    """The module-side conditions of every fused site, local or sync: training mode, tracked running statistics, a
    numeric momentum, and affine weight, bias and running statistics in contiguous fp32."""
    if not bn.training or not bn.track_running_stats or not isinstance(bn.momentum, numbers.Real):
        return False
    return all(t is not None and t.dtype == torch.float32 and t.is_contiguous()
               for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))


def _local_ok(bn, x):
    """_site's conditions of a local training site on the batch norm and its input."""
    local = type(bn) is nn.BatchNorm2d or (isinstance(bn, nn.SyncBatchNorm) and not _torch_syncs(bn))
    if not local or not _module_ok(bn):
        return False
    if not _activation(x) or x.numel() >= 2 ** 31:
        return False
    # one value per channel: torch's batch_norm raises ("Expected more than 1 value per channel"), so must we
    if x.numel() // x.shape[1] <= 1 or not _scratch_bytes(x.shape[1]):
        return False
    return torch._C._select_batch_norm_backend(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, True, bn.eps) == _NATIVE


_PARAM_DTYPES = ({torch.float32}, {torch.bfloat16})


def _infer_bn_ok(bn, x, *operands):
    """_site's conditions of an eval site on the batch norm and its input: `operands` must not require grad either."""
    # eps <= 0 stays on torch, whose F.batch_norm raises for it
    if bn.training or not (type(bn) is nn.BatchNorm2d or isinstance(bn, nn.SyncBatchNorm)) or not bn.eps > 0:
        return False
    params = (bn.weight, bn.bias, bn.running_mean, bn.running_var)
    if any(t is None or not t.is_contiguous() or t.device != x.device for t in params) or {t.dtype for t in params} not in _PARAM_DTYPES:
        return False
    if torch.is_grad_enabled() and any(t.requires_grad for t in (x, bn.weight, bn.bias, *operands)):
        return False
    if not _activation(x) or x.numel() == 0 or x.numel() >= 2 ** 31:
        return False
    return torch._C._select_batch_norm_backend(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, False, bn.eps) == _NATIVE


def _infer_params(bn):
    """weight, bias, running_mean and running_var of an eval site's batch norm, and its param_bf16 flag."""
    return (bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
            int(bn.weight.dtype == torch.bfloat16))


def _infer(bn, x, launch, like=torch.empty_like):
    """The output y of an eval site's one native launch, `like(x)`: like x, or a pooled output (_pooled_like,
    _pooled2_like).  `launch(y, params, stream)` makes the C-ABI call from y's pointer, _infer_params(bn) and the
    current stream."""
    y = like(x)
    N.check(launch(y.data_ptr(), _infer_params(bn), _raw_stream(x.device.index)))
    return y


def _rows(t):
    """_activation, where a tensor without elements (a rank with an empty batch) passes on its device, dtype and rank
    alone: its strides say nothing (a convolution over an empty batch returns default strides whatever its input's
    layout), the kernels read none of its elements, and the sync decision must not depend on a rank's batch size."""
    return _activation(t) or (t.numel() == 0 and t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 4)


def _sync_comm(bn, x):
    """The communicator of a sync site (the conditions of the module docstring), else None.  Only conditions that
    every rank meets alike decide; an input the kernels cannot take raises instead of falling back, since the other
    ranks would wait in this site's collectives."""
    comm = getattr(bn, "b200_comm", None)
    if comm is None or comm.world_size <= 1 or not _module_ok(bn) or not _rows(x):
        return None
    if x.numel() >= 2 ** 31 or not _scratch_bytes(x.shape[1], comm.world_size):
        raise RuntimeError(f"sync batch norm: input of shape {tuple(x.shape)} exceeds the kernels' limits "
                           "(< 2^31 elements, at most 131072 channels)")
    return comm


def _hooked(mod):
    return bool(mod._forward_hooks or mod._forward_pre_hooks or mod._backward_hooks or mod._backward_pre_hooks)


def _global_hooks():
    from torch.nn.modules import module

    return bool(module._global_forward_hooks or module._global_forward_pre_hooks or module._global_backward_hooks
                or module._global_backward_pre_hooks)


def _skips_hooks(*mods):
    """Whether calling kernels in place of the modules `mods` would skip a hook: one of theirs or a global one."""
    return any(map(_hooked, mods)) or _global_hooks()


# how a batch-norm site runs (_site), besides the communicator of a sync site and None for the modules' own ops
_EVAL, _LOCAL = "eval", "local"


def _site(bn, x, mods=(), operands=(), sync=True, inputs=()):
    """How the site of batch norm `bn` on input x runs, by the module docstring's conditions: _EVAL (one launch on the
    eval kernels), _LOCAL (a local training site), the communicator of a sync site, or None: the modules run.  `mods`
    are the other modules whose calls the kernels replace, `operands` the other tensors they read (the identity).
    Where the entry point has no sync form (`sync` False), a sync batch norm gets None and runs its own module forward,
    FusedSyncBatchNorm's sync site.  `inputs` are the tensors x stands for (a concatenation's segments): an eval site
    must not record a gradient for them either."""
    if _skips_hooks(bn, *mods):
        return None
    for t in operands:
        # _rows: an eval or local site has rows, and so then has an operand of x's shape, where _rows is _activation
        if t.shape != x.shape or t.device != x.device or not _rows(t):
            return None
    if _infer_bn_ok(bn, x, *operands, *inputs):
        return _EVAL
    comm = _sync_comm(bn, x)
    if comm is not None:
        return comm if sync else None
    return _LOCAL if _local_ok(bn, x) else None


def bn_relu(bn, relu, x, sync=True):
    """relu(bn(x)), fused when the site allows it.  `relu` None stands for torchvision BasicConv2d's functional
    F.relu(..., inplace=True); with `sync` False a sync batch norm runs its own module forward (FusedSyncBatchNorm's
    sync site) and then the ReLU."""
    site = _site(bn, x, () if relu is None else (relu,), sync=sync) if relu is None or type(relu) is nn.ReLU else None
    if site is _EVAL:
        c = x.shape[1]
        return _infer(bn, x, lambda y, p, s: _native_lib().b200c_bn_infer(x.data_ptr(), None, y, *p, bn.eps, x.numel() // c, c, s))
    if site is not None:
        return _FusedBatchNorm.apply(x, None, bn.weight, bn.bias, bn, False, None if site is _LOCAL else site, True)
    if relu is None:
        return F.relu(bn(x), inplace=True)
    return relu(bn(x))


# the most segments a concatenation site takes (the library's kMaxCatSegs)
_MAX_CAT_SEGS = 64


def _cat_segments_ok(features):
    """Whether a concatenation site can read `features` in place: 1..64 segments, each passing _activation with the
    first one's N, H, W and device, a multiple of 8 channels and a data pointer on the 16-byte grid."""
    if not 1 <= len(features) <= _MAX_CAT_SEGS:
        return False
    f0 = features[0]
    n, _, h, w = f0.shape if f0.dim() == 4 else (None,) * 4
    for t in features:
        if not _activation(t) or t.device != f0.device or t.shape[0] != n or t.shape[2] != h or t.shape[3] != w:
            return False
        if t.shape[1] % 8 or t.data_ptr() % 16:
            return False
    return True


def _cat_table(features):
    """The C-ABI's segment table of `features`: pointers, channels and their count."""
    k = len(features)
    return ((ctypes.c_void_p * k)(*(t.data_ptr() for t in features)), (ctypes.c_int * k)(*(t.shape[1] for t in features)), k)


class _FusedBatchNormCat(torch.autograd.Function):
    """relu(bn(torch.cat(features, 1))) in training mode, reading the segments where they lie: no concatenation is
    written, and the segments themselves (not a copy) are saved for the backward.  The forward writes y and the ReLU's
    mask bits; the backward writes the whole dx once and returns each segment's gradient as the view
    dx.narrow(1, c0, C_s), as torch's CatBackward does, so autograd accumulates each feature map's gradients as it
    would in eager torch."""

    @staticmethod
    def forward(ctx, y, weight, bias, bn, *features):
        # y: the empty output, of the concatenation's shape and layout
        n, c, h, w = y.shape
        m = n * h * w
        mask = torch.empty(m * c // 8, dtype=torch.uint8, device=y.device)
        stats, params, stream, scratch = _forward_args(y, bn, weight, bias)
        N.check(_native_lib().b200c_bn_forward_cat(*_cat_table(features), y.data_ptr(), mask.data_ptr(), *params, m, c, bn.momentum,
                                                   bn.eps, scratch, stream))
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(mask, weight, stats, *features)
        ctx.mark_dirty(y)   # the output buffer the site was decided on, written here
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        mask, weight, stats, *features = ctx.saved_tensors
        if dy is None:
            return (None,) * (4 + len(features))
        dy = dy.contiguous(memory_format=torch.channels_last)
        n, c, h, w = dy.shape
        dx, grad_weight, grad_bias, stream, scratch = _backward_args(dy)
        mean = stats.data_ptr()
        N.check(_native_lib().b200c_bn_backward_cat(dy.data_ptr(), mask.data_ptr(), *_cat_table(features), dx.data_ptr(),
                                                    weight.data_ptr(), mean, mean + 4 * c, grad_weight.data_ptr(),
                                                    grad_bias.data_ptr(), n * h * w, c, scratch, stream))
        grads, c0 = [], 0
        for t in features:
            grads.append(dx.narrow(1, c0, t.shape[1]))
            c0 += t.shape[1]
        return (None, grad_weight, grad_bias, None, *grads)


def bn_relu_cat(bn, relu, features):
    """relu(bn(torch.cat(features, 1))), `relu` an nn.ReLU module or None for the functional F.relu, fused when the
    site allows it: where every segment can be read in place (_cat_segments_ok), the batch norm is decided by `_site`
    on a tensor of the concatenation's shape and layout (the output, allocated first), with the hook rule covering the
    batch norm and the ReLU module, and runs as an eval launch or a local training site over the segments.  Anything
    else, a sync site included, concatenates with torch.cat and runs bn_relu."""
    features = list(features)
    if (relu is None or type(relu) is nn.ReLU) and _cat_segments_ok(features):
        n, _, h, w = features[0].shape
        c = sum(t.shape[1] for t in features)
        y = torch.empty((n, c, h, w), dtype=torch.bfloat16, device=features[0].device, memory_format=torch.channels_last)
        site = _site(bn, y, () if relu is None else (relu,), inputs=features)
        if site is _EVAL:
            N.check(_native_lib().b200c_bn_infer_cat(*_cat_table(features), y.data_ptr(), *_infer_params(bn), bn.eps, n * h * w, c,
                                                     _raw_stream(y.device.index)))
            return y
        if site is _LOCAL:
            return _FusedBatchNormCat.apply(y, bn.weight, bn.bias, bn, *features)
    x = torch.cat(features, 1)
    if relu is None:
        return torch.relu_(bn(x))
    return bn_relu(bn, relu, x)


def _cat_format(tensors):
    """The memory format torch.cat gives its output: the operands' common suggested format, else contiguous."""
    formats = {torch._prims_common.suggest_memory_format(t) for t in tensors}
    return formats.pop() if len(formats) == 1 else torch.contiguous_format


def _slice_operands_ok(tensors):
    """Whether `tensors` (a module's branch outputs, in output order) can be the operands of slice sites: each passes
    _activation with the first one's N, H, W and device, has a multiple of 8 channels (so every slice starts on the
    16-byte grid of the output's rows) and a data pointer on the 16-byte grid, the output has fewer than 2^31 elements,
    and torch.cat would lay it out as rows of channels: channels-last, or either format over one row per sample, where
    both lay out memory alike.  (A channels-last tensor whose strides also fit another order, as N = 1 with W = 1 can
    after a view, may make torch.cat choose the contiguous format.)"""
    t0 = tensors[0]
    if t0.dim() != 4:
        return False
    n, _, h, w = t0.shape
    for t in tensors:
        if not _activation(t) or t.device != t0.device or t.shape[0] != n or t.shape[2] != h or t.shape[3] != w:
            return False
        if t.shape[1] % 8 or t.data_ptr() % 16:
            return False
    if h * w > 1 and _cat_format(tensors) != torch.channels_last:
        return False
    return n * h * w * sum(t.shape[1] for t in tensors) < 2 ** 31


def _concat_like(operands):
    """The empty bf16 output of torch.cat(operands, 1) with the strides torch.cat gives it (_cat_format)."""
    t0 = operands[0]
    n, _, h, w = t0.shape
    return torch.empty((n, sum(t.shape[1] for t in operands), h, w), dtype=torch.bfloat16, device=t0.device,
                       memory_format=_cat_format(operands))


def _rows_of(dy):
    """dy as the slice sites' backward reads it: channels-last with a channel stride of 1 on the 16-byte grid, a copy
    where it arrives otherwise.  The copy is exact: eager torch's threshold_backward writes g in y's layout, which is
    channels-last, whatever the layout of the gradient it is given."""
    if _activation(dy) and dy.data_ptr() % 16 == 0:
        return dy
    return dy.clone(memory_format=torch.channels_last)


class _FusedBatchNormSlices(torch.autograd.Function):
    """torch.cat([relu(bn_b(x_b)) for each site b, or a ready tensor], 1) in training mode: one autograd node for a
    whole Inception module.  `spec` gives, in output order, each branch's batch norm (a site, whose x, weight and bias
    are the next three tensors) or None (a ready tensor, the next one).  Each site writes its output straight into its
    channels of the output and its ReLU's mask bits (b200c_bn_forward_slice); a ready tensor is copied into its
    channels, exactly as torch.cat copies it.  The backward reads each site's channels of dy in place
    (b200c_bn_backward_slice) and returns each ready tensor's gradient as dy.narrow(1, c0, C) of dy as it arrived, which
    is what torch's CatBackward returns, so the ops consuming it (a max-pool backward picks its kernel by layout) see
    what they see in eager torch."""

    @staticmethod
    def forward(ctx, spec, *tensors):
        lib = _native_lib()
        parts, it = [], iter(tensors)
        for bn in spec:
            parts.append((bn, next(it), next(it), next(it)) if bn is not None else (None, next(it), None, None))
        out = _concat_like([x for _, x, _, _ in parts])
        n, ctot, h, w = out.shape
        m = n * h * w
        saved, layout, c0 = [], [], 0
        for bn, x, weight, bias in parts:
            c = x.shape[1]
            if bn is None:
                out.narrow(1, c0, c).copy_(x)
            else:
                mask = torch.empty(m * c // 8, dtype=torch.uint8, device=x.device)
                stats, params, stream, scratch = _forward_args(x, bn, weight, bias)
                N.check(lib.b200c_bn_forward_slice(x.data_ptr(), out.data_ptr() + 2 * c0, ctot, mask.data_ptr(), *params, m, c,
                                                   bn.momentum, bn.eps, scratch, stream))
                saved += [x, mask, weight, stats]
            layout.append((bn is not None, c0, c))
            c0 += c
        ctx.layout = layout
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(*saved)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        layout = ctx.layout
        if dy is None:
            return (None,) + tuple(None for site, _, _ in layout for _ in range(3 if site else 1))
        lib = _native_lib()
        saved = iter(ctx.saved_tensors)
        g = _rows_of(dy)
        ctot = g.shape[1]
        grads = [None]
        for site, c0, c in layout:
            if not site:
                grads.append(dy.narrow(1, c0, c))
                continue
            x, mask, weight, stats = next(saved), next(saved), next(saved), next(saved)
            dx, grad_weight, grad_bias, stream, scratch = _backward_args(x)
            mean = stats.data_ptr()
            N.check(lib.b200c_bn_backward_slice(g.data_ptr() + 2 * c0, ctot, mask.data_ptr(), x.data_ptr(), dx.data_ptr(),
                                                weight.data_ptr(), mean, mean + 4 * c, grad_weight.data_ptr(), grad_bias.data_ptr(),
                                                x.numel() // c, c, scratch, stream))
            grads += [dx, grad_weight, grad_bias]
        return tuple(grads)


def bn_relu_concat(branches):
    """torch.cat(outputs, 1) of a module whose branches, in output order, are each a batch-norm site `(bn, x)` or
    `(bn, x, mods)` standing for F.relu(bn(x), inplace=True) (torchvision's BasicConv2d after its convolution; `mods`
    the other modules whose calls the site replaces), or a ready tensor, with eager torch's bits.  The output is
    allocated once in torch.cat's layout and each site writes its channels of it in place.

    Every site is decided by `_site` (never a sync site), with the ready tensors as inputs an eval site must not record
    a gradient for.  Where every site is an eval site, each runs one b200c_bn_infer_slice launch and each ready tensor
    is copied into its channels; where every site is a local training site, one _FusedBatchNormSlices node runs them
    all.  Anything else (operands _slice_operands_ok refuses, a site that runs its modules, or eval and training sites
    mixed) runs each site's batch norm and ReLU as modules and then torch.cat."""
    sites = [(b[0], b[1], b[2] if len(b) > 2 else ()) for b in branches if isinstance(b, tuple)]
    ready = [b for b in branches if not isinstance(b, tuple)]
    operands = [b[1] if isinstance(b, tuple) else b for b in branches]
    kinds = set()
    if sites and _slice_operands_ok(operands):
        kinds = {_site(bn, x, mods, sync=False, inputs=ready) for bn, x, mods in sites}
    if kinds == {_EVAL}:
        out = _concat_like(operands)
        n, ctot, h, w = out.shape
        m = n * h * w
        lib, stream, c0 = _native_lib(), _raw_stream(out.device.index), 0
        for b in branches:
            if isinstance(b, tuple):
                bn, x = b[0], b[1]
                c = x.shape[1]
                N.check(lib.b200c_bn_infer_slice(x.data_ptr(), out.data_ptr() + 2 * c0, ctot, *_infer_params(bn), bn.eps, m, c, stream))
            else:
                c = b.shape[1]
                out.narrow(1, c0, c).copy_(b)
            c0 += c
        return out
    if kinds == {_LOCAL}:
        spec, tensors = [], []
        for b in branches:
            if isinstance(b, tuple):
                spec.append(b[0])
                tensors += [b[1], b[0].weight, b[0].bias]
            else:
                spec.append(None)
                tensors.append(b)
        return _FusedBatchNormSlices.apply(tuple(spec), *tensors)
    return torch.cat([F.relu(b[0](b[1]), inplace=True) if isinstance(b, tuple) else b for b in branches], 1)


# the most channels a ShuffleNetV2 block end takes per branch: its two-batch-norm form runs in the dual scratch
_MAX_SHUFFLE_CHANNELS = 65536


def _shuffle_operands_ok(x1, sites):
    """Whether a ShuffleNetV2 block end can run on the shuffle kernels: every site's input passes _activation with the
    second one's shape and device, at most 65536 channels, an output of fewer than 2^31 elements, and a ready x1 is
    bf16 of the same shape and device laid out as NCHW planes (what x.chunk(2, 1)[0] of a contiguous x is)."""
    t = sites[-1][1]
    if t.dim() != 4:
        return False
    n, c, h, w = t.shape
    if c > _MAX_SHUFFLE_CHANNELS or 2 * t.numel() >= 2 ** 31:
        return False
    if any(not _activation(x) or x.shape != t.shape or x.device != t.device for _, x, _ in sites):
        return False
    if x1 is None:
        return True
    return (x1.dtype == torch.bfloat16 and x1.device == t.device and x1.shape == t.shape and x1.stride()[1:] == (h * w, w, 1)
            and c * h * w <= x1.stride(0) < 2 ** 31)


def _shuffle_first_grad(dy, b):
    """The gradient eager torch's backward of `channel_shuffle(torch.cat((x1, z), 1), 2)` hands x1 for the output's
    gradient dy: the view/transpose/reshape chain's, narrowed by CatBackward.  Its last reshape copies into a contiguous
    [N, 2B, H, W] tensor unless B == 1 or dy's channel stride is 0 (an expanded gradient), where it is a view of dy; so
    x1's gradient is channels 0..B-1 of such a tensor, of which only those channels are written here."""
    n, _, h, w = dy.shape
    if b == 1 or dy.stride(1) == 0:
        return dy.reshape(n, b, 2, h, w).transpose(1, 2).reshape(n, 2 * b, h, w).narrow(1, 0, b)
    return torch.empty(dy.shape, dtype=dy.dtype, device=dy.device).narrow(1, 0, b).copy_(dy[:, 0::2])


class _FusedBatchNormShuffle(torch.autograd.Function):
    """channel_shuffle(torch.cat((a, relu(bn_t(t))), 1), 2) in training mode, a being x1 (bn_u and u None) or
    relu(bn_u(u)): the end of a ShuffleNetV2 block, one autograd node.  The forward writes the contiguous NCHW output
    and each batch norm's mask bits (b200c_bn_forward_shuffle), never a branch output or the concatenation; the backward
    reads dy channels-last (b200c_bn_backward_shuffle) and gives x1 the gradient eager torch gives it
    (_shuffle_first_grad), values and strides."""

    @staticmethod
    def forward(ctx, bn_t, bn_u, x1, t, weight, bias, u, weight_u, bias_u):
        lib = _native_lib()
        n, c, h, w = t.shape
        m = n * h * w
        two = u is not None
        y = torch.empty((n, 2 * c, h, w), dtype=torch.bfloat16, device=t.device)
        mask_bytes = lib.b200c_bn_shuffle_mask_bytes(m, c)
        mask = torch.empty(mask_bytes, dtype=torch.uint8, device=t.device)
        stats, params, stream, scratch = _forward_args(t, bn_t, weight, bias, dual=two)
        mask_u = stats_u = None
        if two:
            mask_u = torch.empty(mask_bytes, dtype=torch.uint8, device=t.device)
            stats_u, params_u, _, _ = _forward_args(u, bn_u, weight_u, bias_u, dual=True)
            first = (None, 0, u.data_ptr(), mask_u.data_ptr(), *params_u, bn_u.momentum, bn_u.eps)
        else:
            first = (x1.data_ptr(), x1.stride(0), None, None, *(None,) * 7, 0.0, 0.0)
        N.check(lib.b200c_bn_forward_shuffle(*first, t.data_ptr(), mask.data_ptr(), *params, bn_t.momentum, bn_t.eps, y.data_ptr(),
                                             n, h * w, c, scratch, stream))
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(t, mask, weight, stats, u, mask_u, weight_u, stats_u)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        if dy is None:
            return (None,) * 9
        t, mask, weight, stats, u, mask_u, weight_u, stats_u = ctx.saved_tensors
        n, c, h, w = t.shape
        two = u is not None
        g = _rows_of(dy)
        dt, grad_weight, grad_bias, stream, scratch = _backward_args(t, dual=two)
        mean = stats.data_ptr()
        first = (None,) * 8
        if two:
            du, grad_weight_u, grad_bias_u, _, _ = _backward_args(u, dual=True)
            mean_u = stats_u.data_ptr()
            first = (u.data_ptr(), mask_u.data_ptr(), du.data_ptr(), weight_u.data_ptr(), mean_u, mean_u + 4 * c,
                     grad_weight_u.data_ptr(), grad_bias_u.data_ptr())
        N.check(_native_lib().b200c_bn_backward_shuffle(g.data_ptr(), *first, t.data_ptr(), mask.data_ptr(), dt.data_ptr(),
                                                        weight.data_ptr(), mean, mean + 4 * c, grad_weight.data_ptr(),
                                                        grad_bias.data_ptr(), n * h * w, c, scratch, stream))
        if two:
            return None, None, None, dt, grad_weight, grad_bias, du, grad_weight_u, grad_bias_u
        dx1 = _shuffle_first_grad(dy, c) if ctx.needs_input_grad[2] else None
        return None, None, dx1, dt, grad_weight, grad_bias, None, None, None


def bn_relu_shuffle(first, second):
    """channel_shuffle(torch.cat((a, relu(bn(t))), 1), 2), the end of torchvision's ShuffleNetV2 block, with eager torch's
    bits and strides.  `second` is a batch-norm site `(bn, t, mods)`, `first` either one `(bn, u, mods)` (a stride-2
    block's branch1, a = relu(bn(u))) or the ready tensor a = x1 (a stride-1 block's x.chunk(2, 1)[0]); `mods` are the
    other modules whose calls the site replaces, whose hooks `_site` checks.  The output is contiguous NCHW, as
    channel_shuffle's .contiguous() leaves it.

    Every site is decided by `_site` (never a sync site), with x1 among the inputs an eval site must not record a
    gradient for.  Where every site is an eval site the block end is one b200c_bn_infer_shuffle launch; where every site
    is a local training site, one _FusedBatchNormShuffle node.  Anything else (operands _shuffle_operands_ok refuses, a
    site that runs its modules, or eval and training mixed) runs the batch norms and ReLUs as modules, torch.cat and
    torchvision's channel_shuffle."""
    sites = [first, second] if isinstance(first, tuple) else [second]
    x1 = None if isinstance(first, tuple) else first
    kinds = set()
    if _shuffle_operands_ok(x1, sites):
        kinds = {_site(bn, x, mods, sync=False, inputs=() if x1 is None else (x1,)) for bn, x, mods in sites}
    bn_t, t = second[0], second[1]
    bn_u, u = (first[0], first[1]) if x1 is None else (None, None)
    if kinds == {_EVAL} and (u is None or bn_u.weight.dtype == bn_t.weight.dtype):
        n, c, h, w = t.shape
        y = torch.empty((n, 2 * c, h, w), dtype=torch.bfloat16, device=t.device)
        p = _infer_params(bn_t)
        if u is None:
            lead = (x1.data_ptr(), x1.stride(0), None, None, None, None, None, 0.0)
        else:
            lead = (None, 0, u.data_ptr(), *_infer_params(bn_u)[:4], bn_u.eps)
        N.check(_native_lib().b200c_bn_infer_shuffle(*lead, t.data_ptr(), *p[:4], bn_t.eps, y.data_ptr(), p[4], n, h * w, c,
                                                     _raw_stream(t.device.index)))
        return y
    if kinds == {_LOCAL}:
        if u is None:
            return _FusedBatchNormShuffle.apply(bn_t, None, x1, t, bn_t.weight, bn_t.bias, None, None, None)
        return _FusedBatchNormShuffle.apply(bn_t, bn_u, None, t, bn_t.weight, bn_t.bias, u, bn_u.weight, bn_u.bias)
    from torchvision.models.shufflenetv2 import channel_shuffle

    a = x1 if u is None else F.relu(bn_u(u), inplace=True)
    return channel_shuffle(torch.cat((a, F.relu(bn_t(t), inplace=True)), 1), 2)


# activations with native batch-norm sites of their own, by their b200c_act_t (ReLU runs on bn_relu's sites)
_ACT_CODES = {nn.ReLU6: N.ACT_RELU6, nn.SiLU: N.ACT_SILU, nn.Hardswish: N.ACT_HARDSWISH}


def bn_act(bn, act, x):
    """act(bn(x)) for `act` an nn.ReLU, nn.ReLU6, nn.SiLU or nn.Hardswish (exactly those classes), fused when the site
    allows it: ReLU through bn_relu (its sync sites included); for the others an eval site, else a local training
    site.  A sync site with another activation runs the batch norm's own forward (FusedSyncBatchNorm's sync site) and
    then `act`; anything else runs `act(bn(x))`."""
    if type(act) is nn.ReLU:
        return bn_relu(bn, act, x)
    code = _ACT_CODES.get(type(act))
    site = _site(bn, x, (act,), sync=False) if code is not None else None
    if site is _EVAL:
        c = x.shape[1]
        return _infer(bn, x, lambda y, p, s: _native_lib().b200c_bn_infer_act(x.data_ptr(), y, *p, bn.eps, code, x.numel() // c, c, s))
    if site is _LOCAL:
        return _FusedBatchNormAct.apply(x, bn.weight, bn.bias, bn, code)
    return act(bn(x))


def _noise_ok(noise, x):
    """Whether `noise` is stochastic depth's "row" noise for `x` as the kernels read it: bf16 [N, 1, 1, 1] on x's device."""
    return (noise.dtype == torch.bfloat16 and noise.device == x.device and noise.shape == (x.shape[0], 1, 1, 1)
            and noise.is_contiguous() and not noise.requires_grad)


def bn_res(bn, x, identity=None, noise=None):
    """`bn(x)`, `bn(x) + identity`, or with `noise` (torchvision's stochastic depth noise in "row" mode, [N, 1, 1, 1])
    `bn(x) * noise + identity`, with eager torch's bits, fused when the site allows it: an eval site (no noise) in one
    launch, else a local training site.  Noise needs an identity.  Anything else runs the modules' ops."""
    site = None
    if noise is None or (identity is not None and _noise_ok(noise, x)):
        site = _site(bn, x, operands=() if identity is None else (identity,), sync=False)
    if site is _EVAL and noise is None:
        c = x.shape[1]
        id_ptr = identity.data_ptr() if identity is not None else None
        return _infer(bn, x, lambda y, p, s: _native_lib().b200c_bn_infer_res(x.data_ptr(), id_ptr, y, *p, bn.eps, x.numel() // c, c, s))
    if site is _LOCAL:
        return _FusedBatchNormRes.apply(x, identity, bn.weight, bn.bias, bn, noise)
    out = bn(x)
    if noise is not None:
        out = out * noise
    return out if identity is None else out + identity


def _pool_fusable(pool):
    """Whether the stem kernel can replace `pool`'s call: `pool` is exactly nn.MaxPool2d(3, 2, 1) (dilation 1, floor
    mode, no indices) without a hook of its own (the site's `_site` checks the global ones)."""
    two = lambda v, k: v in (k, (k, k))  # noqa: E731
    return (type(pool) is nn.MaxPool2d and two(pool.kernel_size, 3) and two(pool.stride, 2) and two(pool.padding, 1)
            and two(pool.dilation, 1) and not pool.ceil_mode and not pool.return_indices and not _hooked(pool))


def _pool2_fusable(pool):
    """Whether the VGG stage-end kernels can replace `pool`'s call: `pool` is exactly nn.MaxPool2d(2, 2) (padding 0,
    dilation 1, floor mode, no indices) without a hook of its own (the site's `_site` checks the global ones)."""
    two = lambda v, k: v in (k, (k, k))  # noqa: E731
    return (type(pool) is nn.MaxPool2d and two(pool.kernel_size, 2) and two(pool.stride, 2) and two(pool.padding, 0)
            and two(pool.dilation, 1) and not pool.ceil_mode and not pool.return_indices and not _hooked(pool))


def bn_relu_maxpool(bn, relu, pool, x):
    """pool(relu(bn(x))), fused into one site when `pool` is nn.MaxPool2d(3, 2, 1) (the ResNet stem) or nn.MaxPool2d(2,
    2) (a VGG stage end) and the batch norm can run as an eval or a local training site; otherwise bn_relu and the
    module call."""
    site = _site(bn, x, (relu,), sync=False) if type(relu) is nn.ReLU and _pool_fusable(pool) else None
    if site is _EVAL:
        n, c, h, w = x.shape
        return _infer(bn, x, lambda y, p, s: _native_lib().b200c_bn_infer_pool(x.data_ptr(), y, *p, bn.eps, n, h, w, c, s),
                      like=_pooled_like)
    if site is _LOCAL:
        return _FusedBatchNormPool.apply(x, bn.weight, bn.bias, bn)
    # VGG's stage end; an h or w below 2 is left to torch's max_pool2d, which raises for it
    site = None
    if type(relu) is nn.ReLU and _pool2_fusable(pool) and x.dim() == 4 and min(x.shape[2:]) >= 2:
        site = _site(bn, x, (relu,), sync=False)
    if site is _EVAL:
        n, c, h, w = x.shape
        return _infer(bn, x, lambda y, p, s: _native_lib().b200c_bn_infer_pool2(x.data_ptr(), y, *p, bn.eps, n, h, w, c, s),
                      like=_pooled2_like)
    if site is _LOCAL:
        return _FusedBatchNormPool2.apply(x, bn.weight, bn.bias, bn)
    return pool(bn_relu(bn, relu, x))


def bn_add_relu(bn, relu, x, identity, pair=False):
    """`out = bn(x); out += identity; relu(out)`, fused when the site allows it.  With `pair`, returns `(out,
    out_id)`: the same values, whose gradients a fused site receives apart and sums in its backward kernel."""
    site = _site(bn, x, (relu,), (identity,)) if type(relu) is nn.ReLU else None
    if site is _EVAL:
        c = x.shape[1]
        out = _infer(bn, x, lambda y, p, s: _native_lib().b200c_bn_infer(x.data_ptr(), identity.data_ptr(), y, *p, bn.eps,
                                                                          x.numel() // c, c, s))
        return (out, out) if pair else out
    if site is not None:
        return _FusedBatchNorm.apply(x, identity, bn.weight, bn.bias, bn, pair, None if site is _LOCAL else site, True)
    out = bn(x)
    out += identity
    out = relu(out)
    return (out, out) if pair else out


def _downsample_bn(ds):
    """The batch norm of a downsample branch that a dual tail can run: `ds` exactly nn.Sequential(nn.Conv2d, batch
    norm), neither the Sequential nor the batch norm with a hook of its own (the site's `_site` checks the global
    ones); else None."""
    if type(ds) is not nn.Sequential or len(ds) != 2 or type(ds[0]) is not nn.Conv2d or _hooked(ds) or _hooked(ds[1]):
        return None
    return ds[1]


def bn_add_relu_downsample(bn, relu, x, downsample, x_id, pair=False):
    """`out = bn(x); out += downsample(x_id); relu(out)`, with `pair` as in bn_add_relu.  Where the downsample branch is
    a convolution and a batch norm that can run as a local fused site alongside this one, both batch norms run in
    one native call per direction (in eval, one launch) and the branch's output is never written; otherwise
    bn_add_relu."""
    bn_ds = _downsample_bn(downsample)
    site = None
    if bn_ds is not None and bn_ds is not bn and type(relu) is nn.ReLU:
        site = _site(bn, x, (relu,), sync=False)
    if site is None:
        return bn_add_relu(bn, relu, x, downsample(x_id), pair)
    x_ds = downsample[0](x_id)
    site_ds = _site(bn_ds, x_ds, sync=False) if x_ds.shape == x.shape else None
    if site is _EVAL and site_ds is _EVAL and bn_ds.weight.dtype == bn.weight.dtype:
        c = x.shape[1]
        out = _infer(bn, x, lambda y, p, s: _native_lib().b200c_bn_infer_dual(
            x.data_ptr(), x_ds.data_ptr(), y, *p[:4], bn.eps, *_infer_params(bn_ds)[:4], bn_ds.eps, p[4], x.numel() // c, c, s))
        return (out, out) if pair else out
    if site is _LOCAL and site_ds is _LOCAL and _scratch_bytes(x.shape[1], "dual"):
        return _FusedBatchNormDual.apply(x, x_ds, bn.weight, bn.bias, bn_ds.weight, bn_ds.bias, bn, bn_ds, pair)
    return bn_add_relu(bn, relu, x, bn_ds(x_ds), pair)


try:
    from torchvision.models.resnet import BasicBlock, Bottleneck, ResNet
except ImportError:  # without torchvision there is nothing to rewrite
    _SWAP = {}
else:

    # A block's input x feeds conv1 and the identity branch.  forward_pair(x, x_id) -> (out, out_id) takes the two
    # as separate tensors and returns its output twice, so that chained blocks hand each tail's backward the two
    # gradients of its output apart, to be summed inside the kernel instead of by a separate add.

    # In eval mode without autograd recording the same helpers run each site on the eval kernels (one launch per
    # site); with autograd recording, eval keeps the parent class's ops.

    class FusedBasicBlock(BasicBlock):
        def forward(self, x):
            if not self.training and torch.is_grad_enabled():
                return super().forward(x)
            return self.forward_pair(x, x)[0]

        def forward_pair(self, x, x_id):
            out = bn_relu(self.bn1, self.relu, self.conv1(x))
            out = self.conv2(out)
            if self.downsample is not None:
                return bn_add_relu_downsample(self.bn2, self.relu, out, self.downsample, x_id, pair=True)
            return bn_add_relu(self.bn2, self.relu, out, x_id, pair=True)

    class FusedBottleneck(Bottleneck):
        def forward(self, x):
            if not self.training and torch.is_grad_enabled():
                return super().forward(x)
            return self.forward_pair(x, x)[0]

        def forward_pair(self, x, x_id):
            out = bn_relu(self.bn1, self.relu, self.conv1(x))
            out = bn_relu(self.bn2, self.relu, self.conv2(out))
            out = self.conv3(out)
            if self.downsample is not None:
                return bn_add_relu_downsample(self.bn3, self.relu, out, self.downsample, x_id, pair=True)
            return bn_add_relu(self.bn3, self.relu, out, x_id, pair=True)

    def _pairwise(layer):
        """Whether `layer`'s blocks can be chained through forward_pair: a plain Sequential of fused blocks, where
        calling forward_pair directly skips no module hook."""
        return (type(layer) is nn.Sequential and not _hooked(layer)
                and all(type(b) in (FusedBasicBlock, FusedBottleneck) and not _hooked(b) for b in layer))

    class FusedResNet(ResNet):
        def forward(self, x):
            if not self.training and torch.is_grad_enabled():
                return super().forward(x)
            x = x_id = bn_relu_maxpool(self.bn1, self.relu, self.maxpool, self.conv1(x))   # two gradients, summed by autograd
            hooks = _global_hooks()
            for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
                if self.training and not hooks and _pairwise(layer):
                    for block in layer:
                        x, x_id = block.forward_pair(x, x_id)
                else:
                    x = x_id = layer(x)
            x = torch.flatten(self.avgpool(x), 1)
            return self.fc(x)

    _SWAP = {ResNet: FusedResNet, Bottleneck: FusedBottleneck, BasicBlock: FusedBasicBlock}


class FusedSyncBatchNorm(nn.SyncBatchNorm):
    """nn.SyncBatchNorm whose sync sites run on the peer-memory communicator `b200_comm` (see `sync_batch_norm`).
    Its own forward is a site with nothing fused after it; anything that is not a sync site runs nn.SyncBatchNorm's
    forward unchanged."""

    b200_comm = None

    def forward(self, x):
        # _site's sync step alone: the module call has run this module's hooks and replaces no other module, and this
        # is where every other site with a sync batch norm that runs its modules joins the collectives
        comm = _sync_comm(self, x)
        if comm is None:
            return super().forward(x)
        return _FusedBatchNorm.apply(x, None, self.weight, self.bias, self, False, comm, False)


def _world_group(pg):
    return pg is None or (dist.is_available() and dist.is_initialized() and pg == dist.group.WORLD)


def has_world_sync_batch_norm(model):
    """Whether `model` has an nn.SyncBatchNorm over the world group (process_group None or WORLD)."""
    return any(isinstance(m, nn.SyncBatchNorm) and _world_group(m.process_group) for m in model.modules())


def sync_batch_norm(model, comm):
    """Rewrite `model` in place: every nn.SyncBatchNorm (exactly that class, or FusedSyncBatchNorm) over the world
    group becomes a FusedSyncBatchNorm that runs its sync sites over `comm`, a PeerMemoryComm of the same ranks.
    Parameters, buffers, state_dict keys, hooks and the object itself are unchanged.  SyncBatchNorm over a process
    subgroup is left to torch."""
    for mod in model.modules():
        if type(mod) in (nn.SyncBatchNorm, FusedSyncBatchNorm) and _world_group(mod.process_group):
            mod.__class__ = FusedSyncBatchNorm
            mod.b200_comm = comm
    return model


try:
    from torchvision.ops.misc import Conv2dNormActivation
except ImportError:  # without torchvision there is nothing to rewrite
    Conv2dNormActivation = None
else:

    class FusedConv2dNormActivation(Conv2dNormActivation):
        """torchvision's Conv2dNormActivation whose batch norm and activation run as one site (`bn_act`) when the block
        is exactly an nn.Conv2d, a BatchNorm2d or SyncBatchNorm, and an nn.ReLU6, SiLU or Hardswish, and calling the
        kernels instead of those two modules skips no hook.  The convolution is still called as a module, and the
        block's own hooks run as before.  Anything else, and eval with gradients recorded, runs the parent's forward."""

        def forward(self, x):
            if len(self) != 3 or (not self.training and torch.is_grad_enabled()):
                return super().forward(x)
            conv, bn, act = self[0], self[1], self[2]
            if (type(conv) is not nn.Conv2d or not (type(bn) is nn.BatchNorm2d or isinstance(bn, nn.SyncBatchNorm))
                    or type(act) not in _ACT_CODES):
                return super().forward(x)
            return bn_act(bn, act, conv(x))


def _row_noise(sd, t):
    """torchvision's stochastic_depth(t, sd.p, "row", sd.training) noise, built by the same torch calls in the same
    order (so the RNG stream and the bits are torch's), or None where it returns t unchanged (eval, p == 0)."""
    if not sd.training or sd.p == 0.0:
        return None
    survival_rate = 1.0 - sd.p
    noise = torch.empty([t.shape[0]] + [1] * (t.ndim - 1), dtype=t.dtype, device=t.device)
    noise = noise.bernoulli_(survival_rate)
    if survival_rate > 0.0:
        noise.div_(survival_rate)
    return noise


def _res_forward(block, seq, nested, x, identity, sd=None):
    """The inverted-residual block's forward with its projection batch norm as one bn_res site: every module of `seq`
    before the projection, then the projection's convolution as a module, then bn_res with `identity` (None without a
    residual connection) and stochastic depth `sd`'s noise.  The projection is `seq`'s last two modules, or with
    `nested` the two of its last module, a Conv2dNormActivation without activation.

    None where the block must run its parent's forward: eval with gradients recorded, a projection other than exactly
    nn.Conv2d then nn.BatchNorm2d (a SyncBatchNorm stays with FusedSyncBatchNorm), stochastic depth other than
    torchvision's in "row" mode with 0 <= p <= 1, or a hook that calling the modules one by one would skip (on `seq`,
    the projection's Conv2dNormActivation, the batch norm, `sd`, or a global one)."""
    if (not block.training and torch.is_grad_enabled()) or type(seq) is not nn.Sequential or len(seq) < 2:
        return None
    if nested:
        last = seq[-1]
        if type(last) is not Conv2dNormActivation or len(last) != 2:
            return None
        head, conv, bn, mods = list(seq)[:-1], last[0], last[1], [seq, last]
    else:
        head, conv, bn, mods = list(seq)[:-2], seq[-2], seq[-1], [seq]
    if type(conv) is not nn.Conv2d or type(bn) is not nn.BatchNorm2d:
        return None
    if sd is not None:
        if type(sd) is not StochasticDepth or sd.mode != "row" or not 0.0 <= sd.p <= 1.0:
            return None
        mods.append(sd)
    if _skips_hooks(bn, *mods):
        return None
    out = x
    for mod in head:
        out = mod(out)
    out = conv(out)
    noise = _row_noise(sd, out) if sd is not None and identity is not None else None
    return bn_res(bn, out, identity, noise)


try:
    from torchvision.models import efficientnet, mobilenetv2, mobilenetv3
    from torchvision.ops import StochasticDepth
except ImportError:  # without torchvision there is nothing to rewrite
    _RES_SWAP = {}
else:

    # The projection of these blocks ends in an nn.Conv2d and a batch norm without activation: MobileNetV2's last two
    # modules of `conv`, MobileNetV3's and EfficientNet's last Conv2dNormActivation of `block` (activation_layer None).

    class FusedInvertedResidualV2(mobilenetv2.InvertedResidual):
        """MobileNetV2's block, `x + conv(x)` or `conv(x)`, whose projection batch norm and residual add are one bn_res site."""

        def forward(self, x):
            out = _res_forward(self, self.conv, False, x, x if self.use_res_connect else None)
            return super().forward(x) if out is None else out

    class FusedInvertedResidualV3(mobilenetv3.InvertedResidual):
        """MobileNetV3's block, `block(x)` then `+= x`, whose projection batch norm and residual add are one bn_res site."""

        def forward(self, input):
            out = _res_forward(self, self.block, True, input, input if self.use_res_connect else None)
            return super().forward(input) if out is None else out

    class FusedMBConv(efficientnet.MBConv):
        """EfficientNet's block, `stochastic_depth(block(x))` then `+= x`, whose projection batch norm, stochastic depth
        and residual add are one bn_res site."""

        def forward(self, input):
            out = _res_forward(self, self.block, True, input, input if self.use_res_connect else None,
                               self.stochastic_depth)
            return super().forward(input) if out is None else out

    _RES_SWAP = {mobilenetv2.InvertedResidual: FusedInvertedResidualV2, mobilenetv3.InvertedResidual: FusedInvertedResidualV3,
                 efficientnet.MBConv: FusedMBConv}


try:
    from torchvision.models import densenet
except ImportError:  # without torchvision there is nothing to rewrite
    _DENSE_SWAP = {}
else:

    class FusedDenseLayer(densenet._DenseLayer):
        """torchvision's dense layer whose `relu1(norm1(torch.cat(features, 1)))` is one concatenation site
        (`bn_relu_cat`) that reads the earlier feature maps in place, and whose norm2 / relu2 is a bn_relu site; the
        convolutions and the dropout run as torchvision runs them.  Where torchvision would checkpoint the bottleneck
        (`memory_efficient` with a gradient needed), and in eval with gradients recorded, the parent's forward runs."""

        def forward(self, input):
            prev = [input] if isinstance(input, torch.Tensor) else input
            if (self.memory_efficient and self.any_requires_grad(prev)) or (not self.training and torch.is_grad_enabled()):
                return super().forward(input)
            out = self.conv1(bn_relu_cat(self.norm1, self.relu1, prev))
            out = self.conv2(bn_relu(self.norm2, self.relu2, out))
            if self.drop_rate > 0:
                out = F.dropout(out, p=self.drop_rate, training=self.training)
            return out

    class FusedDenseBlock(densenet._DenseBlock):
        """torchvision's dense block, with `forward_features`: the list of feature maps its forward would concatenate."""

        def forward_features(self, init_features):
            """[init_features, each layer's output]: the layers called as torchvision's forward calls them, without the
            final torch.cat."""
            features = [init_features]
            for _, layer in self.items():
                features.append(layer(features))
            return features

    def _dense_walk(features):
        """The (block, transition or None) pairs of a DenseNet's `features` that FusedDenseNet.forward walks: `features`
        an nn.Sequential of exactly conv0, norm0, relu0, pool0, then FusedDenseBlocks and torchvision _Transitions
        (norm, relu, conv, pool) in turn, ending in a block and norm5, where neither `features` nor a block or
        transition has a hook of its own (calling their parts skips their calls); else None."""
        if type(features) is not nn.Sequential or _hooked(features):
            return None
        names, mods = zip(*features.named_children()) if len(features) else ((), ())
        if names[:4] != ("conv0", "norm0", "relu0", "pool0") or names[-1] != "norm5" or len(names) % 2:
            return None
        body = mods[4:-1]
        for i, mod in enumerate(body):
            if type(mod) is not (FusedDenseBlock if i % 2 == 0 else densenet._Transition) or _hooked(mod):
                return None
            if i % 2 and tuple(k for k, _ in mod.named_children()) != ("norm", "relu", "conv", "pool"):
                return None
        return [(body[i], body[i + 1] if i + 1 < len(body) else None) for i in range(0, len(body), 2)]

    class FusedDenseNet(densenet.DenseNet):
        """torchvision's DenseNet whose forward skips the concatenations: the stem is one bn_relu_maxpool site, each
        block hands its transition (or norm5) the list of its feature maps, and each transition's norm / relu and
        norm5 with DenseNet's functional ReLU are concatenation sites (`bn_relu_cat`).  Where `_dense_walk` finds no
        walk, a global module hook is registered, or in eval with gradients recorded, the parent's forward runs (whose
        dense layers still fuse)."""

        def forward(self, x):
            walk = None if not self.training and torch.is_grad_enabled() else _dense_walk(self.features)
            if walk is None or _global_hooks():
                return super().forward(x)
            f = self.features
            x = bn_relu_maxpool(f.norm0, f.relu0, f.pool0, f.conv0(x))
            for block, transition in walk:
                features = block.forward_features(x)
                if transition is not None:
                    x = transition.pool(transition.conv(bn_relu_cat(transition.norm, transition.relu, features)))
            out = bn_relu_cat(f.norm5, None, features)
            out = torch.flatten(F.adaptive_avg_pool2d(out, (1, 1)), 1)
            return self.classifier(out)

    _DENSE_SWAP = {densenet._DenseLayer: FusedDenseLayer, densenet._DenseBlock: FusedDenseBlock, densenet.DenseNet: FusedDenseNet}


try:
    import importlib

    # torchvision.models re-exports the builder functions under the modules' names, so the modules come from importlib
    _inception = importlib.import_module("torchvision.models.inception")
    _googlenet = importlib.import_module("torchvision.models.googlenet")
except ImportError:  # without torchvision there is nothing to rewrite
    _SLICE_SWAP = {}
else:

    def _basic_conv_forward(self, x):
        return bn_relu(self.bn, None, self.conv(x), sync=False)

    class FusedInceptionBasicConv2d(_inception.BasicConv2d):
        """Inception3's BasicConv2d, `F.relu(bn(conv(x)), inplace=True)`, whose batch norm and ReLU run as a bn_relu eval
        or local site; a sync batch norm, or anything else, runs the module ops."""

        forward = _basic_conv_forward

    class FusedGoogLeNetBasicConv2d(_googlenet.BasicConv2d):
        """GoogLeNet's BasicConv2d, as FusedInceptionBasicConv2d."""

        forward = _basic_conv_forward

    _BASIC_CONVS = (FusedInceptionBasicConv2d, FusedGoogLeNetBasicConv2d)

    def _tail(blk, x, *mods):
        """The slice site of a branch's last block `blk` on its input x: its convolution called as a module, then
        bn_relu_concat's site for its batch norm and ReLU.  `mods` are the other modules whose calls the site replaces
        (a GoogLeNet branch's Sequential)."""
        return (blk.bn, blk.conv(x), (blk, *mods))

    def _seq_tail(seq, x):
        """The slice site of a GoogLeNet branch Sequential: every module but the last called in turn, then _tail."""
        for mod in list(seq)[:-1]:
            x = mod(x)
        return _tail(seq[-1], x, seq)

    def _slice_forward(module, tails, seqs, branches):
        """An Inception module's output from `branches()`, its branch outputs in output order as bn_relu_concat takes
        them, or None where the parent's forward must run: eval with gradients recorded, a branch-ending block `tails`
        that is not a fused BasicConv2d, or a hook that the bypassed calls would skip (on a tail, its batch norm, a
        branch Sequential of `seqs`, or a global one).  branches() calls every convolution in torchvision's order and
        leaves each branch's last batch norm to bn_relu_concat, after all of them: so the backward runs each branch's
        chain in eager torch's order, and the module input's gradient, a bf16 sum over the branches, adds them in eager
        torch's order."""
        if not module.training and torch.is_grad_enabled():
            return None
        if any(type(t) not in _BASIC_CONVS for t in tails) or _skips_hooks(*tails, *(t.bn for t in tails), *seqs):
            return None
        return bn_relu_concat(branches())

    def _avg_pool(x):
        return F.avg_pool2d(x, kernel_size=3, stride=1, padding=1)

    def _max_pool(x):
        return F.max_pool2d(x, kernel_size=3, stride=2)

    class FusedInceptionA(_inception.InceptionA):
        """Inception3's InceptionA whose four branches end in slice sites of one output (bn_relu_concat)."""

        def forward(self, x):
            out = _slice_forward(self, (self.branch1x1, self.branch5x5_2, self.branch3x3dbl_3, self.branch_pool), (), lambda: [
                _tail(self.branch1x1, x),
                _tail(self.branch5x5_2, self.branch5x5_1(x)),
                _tail(self.branch3x3dbl_3, self.branch3x3dbl_2(self.branch3x3dbl_1(x))),
                _tail(self.branch_pool, _avg_pool(x)),
            ])
            return super().forward(x) if out is None else out

    class FusedInceptionB(_inception.InceptionB):
        """Inception3's InceptionB: two slice sites and the max-pool branch as a ready tensor."""

        def forward(self, x):
            out = _slice_forward(self, (self.branch3x3, self.branch3x3dbl_3), (), lambda: [
                _tail(self.branch3x3, x),
                _tail(self.branch3x3dbl_3, self.branch3x3dbl_2(self.branch3x3dbl_1(x))),
                _max_pool(x),
            ])
            return super().forward(x) if out is None else out

    class FusedInceptionC(_inception.InceptionC):
        """Inception3's InceptionC whose four branches end in slice sites of one output."""

        def forward(self, x):
            out = _slice_forward(self, (self.branch1x1, self.branch7x7_3, self.branch7x7dbl_5, self.branch_pool), (), lambda: [
                _tail(self.branch1x1, x),
                _tail(self.branch7x7_3, self.branch7x7_2(self.branch7x7_1(x))),
                _tail(self.branch7x7dbl_5, self.branch7x7dbl_4(self.branch7x7dbl_3(self.branch7x7dbl_2(self.branch7x7dbl_1(x))))),
                _tail(self.branch_pool, _avg_pool(x)),
            ])
            return super().forward(x) if out is None else out

    class FusedInceptionD(_inception.InceptionD):
        """Inception3's InceptionD: two slice sites and the max-pool branch as a ready tensor."""

        def forward(self, x):
            out = _slice_forward(self, (self.branch3x3_2, self.branch7x7x3_4), (), lambda: [
                _tail(self.branch3x3_2, self.branch3x3_1(x)),
                _tail(self.branch7x7x3_4, self.branch7x7x3_3(self.branch7x7x3_2(self.branch7x7x3_1(x)))),
                _max_pool(x),
            ])
            return super().forward(x) if out is None else out

    class FusedInceptionE(_inception.InceptionE):
        """Inception3's InceptionE, whose inner concatenations flatten into the outer one: six slice sites, 2a / 2b and
        3a / 3b at their final offsets."""

        def forward(self, x):
            def branches():
                b1 = _tail(self.branch1x1, x)
                t = self.branch3x3_1(x)
                b2a, b2b = _tail(self.branch3x3_2a, t), _tail(self.branch3x3_2b, t)
                t = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
                b3a, b3b = _tail(self.branch3x3dbl_3a, t), _tail(self.branch3x3dbl_3b, t)
                return [b1, b2a, b2b, b3a, b3b, _tail(self.branch_pool, _avg_pool(x))]

            tails = (self.branch1x1, self.branch3x3_2a, self.branch3x3_2b, self.branch3x3dbl_3a, self.branch3x3dbl_3b, self.branch_pool)
            out = _slice_forward(self, tails, (), branches)
            return super().forward(x) if out is None else out

    class FusedInception(_googlenet.Inception):
        """GoogLeNet's Inception module whose four branches end in slice sites of one output; the Sequentials of
        branches 2 to 4 are walked module by module."""

        def forward(self, x):
            seqs = (self.branch2, self.branch3, self.branch4)
            out = None
            if all(type(s) is nn.Sequential and len(s) > 0 for s in seqs):
                out = _slice_forward(self, (self.branch1, *(s[-1] for s in seqs)), seqs, lambda: [
                    _tail(self.branch1, x), _seq_tail(self.branch2, x), _seq_tail(self.branch3, x), _seq_tail(self.branch4, x),
                ])
            return super().forward(x) if out is None else out

    _SLICE_SWAP = {_inception.BasicConv2d: FusedInceptionBasicConv2d, _googlenet.BasicConv2d: FusedGoogLeNetBasicConv2d,
                   _inception.InceptionA: FusedInceptionA, _inception.InceptionB: FusedInceptionB,
                   _inception.InceptionC: FusedInceptionC, _inception.InceptionD: FusedInceptionD,
                   _inception.InceptionE: FusedInceptionE, _googlenet.Inception: FusedInception}


try:
    from torchvision.models import shufflenetv2
except ImportError:  # without torchvision there is nothing to rewrite
    _SHUFFLE_SWAP = {}
else:

    _BN_CLASSES = (nn.BatchNorm2d, nn.SyncBatchNorm)

    def _is_seq(seq, classes):
        """Whether `seq` is exactly an nn.Sequential of modules of `classes`, in order (a batch norm BatchNorm2d or
        SyncBatchNorm)."""
        if type(seq) is not nn.Sequential or len(seq) != len(classes):
            return False
        return all(isinstance(m, _BN_CLASSES) if cls is nn.BatchNorm2d else type(m) is cls for m, cls in zip(seq, classes))

    # torchvision's branches: branch1 (stride 2) depthwise conv, bn, 1x1 conv, bn, ReLU; branch2 1x1 conv, bn, ReLU,
    # depthwise conv, bn, 1x1 conv, bn, ReLU
    _BRANCH1 = (nn.Conv2d, nn.BatchNorm2d, nn.Conv2d, nn.BatchNorm2d, nn.ReLU)
    _BRANCH2 = (nn.Conv2d, nn.BatchNorm2d, nn.ReLU, nn.Conv2d, nn.BatchNorm2d, nn.Conv2d, nn.BatchNorm2d, nn.ReLU)

    def _shuffle_forward(block, x):
        """A ShuffleNetV2 block's output with its branches walked module by module and its end one bn_relu_shuffle, or
        None where the parent's forward must run: eval with gradients recorded, a branch that is not exactly
        torchvision's, or a hook that the walk would skip (on a branch Sequential, a tail batch norm or its ReLU, or a
        global one).  Every module the walk calls runs its own hooks."""
        if not block.training and torch.is_grad_enabled():
            return None
        b1, b2 = block.branch1, block.branch2
        if not _is_seq(b2, _BRANCH2) or not _is_seq(b1, _BRANCH1 if block.stride > 1 else ()):
            return None
        tails = (b2, b2[6], b2[7]) + ((b1, b1[3], b1[4]) if block.stride > 1 else ())
        if _skips_hooks(*tails):
            return None
        if block.stride == 1:
            x1, x2 = x.chunk(2, dim=1)
            first = x1
        else:
            x2 = x
            first = (b1[3], b1[2](bn_res(b1[1], b1[0](x))), (b1[4], b1))
        out = bn_relu(b2[1], b2[2], b2[0](x2))
        out = b2[5](bn_res(b2[4], b2[3](out)))
        return bn_relu_shuffle(first, (b2[6], out, (b2[7], b2)))

    class FusedShuffleInvertedResidual(shufflenetv2.InvertedResidual):
        """ShuffleNetV2's block whose branches run module by module: each first batch norm and ReLU of branch2 a bn_relu
        site, each batch norm after a depthwise convolution a bn_res site, and the branch ends with torch.cat and
        channel_shuffle one bn_relu_shuffle site that writes the shuffled output directly."""

        def forward(self, x):
            out = _shuffle_forward(self, x)
            return super().forward(x) if out is None else out

    def _stem_ok(seq):
        """Whether ShuffleNetV2's conv1 or conv5 `seq` is exactly nn.Sequential(Conv2d, batch norm, ReLU) with no hook on
        it or its parts."""
        return _is_seq(seq, (nn.Conv2d, nn.BatchNorm2d, nn.ReLU)) and not any(map(_hooked, (seq, *seq)))

    class FusedShuffleNetV2(shufflenetv2.ShuffleNetV2):
        """ShuffleNetV2 whose conv1, batch norm, ReLU and max-pool stem is one bn_relu_maxpool site and whose conv5 batch
        norm and ReLU is a bn_relu site; the stages, the mean and fc run as torchvision runs them.  Hooks on conv1,
        conv5 or their parts, a global hook, and eval with gradients recorded run the parent's forward (whose blocks
        still fuse)."""

        def forward(self, x):
            if (not self.training and torch.is_grad_enabled()) or not (_stem_ok(self.conv1) and _stem_ok(self.conv5)) or _global_hooks():
                return super().forward(x)
            c1, c5 = self.conv1, self.conv5
            x = bn_relu_maxpool(c1[1], c1[2], self.maxpool, c1[0](x))
            x = self.stage4(self.stage3(self.stage2(x)))
            x = bn_relu(c5[1], c5[2], c5[0](x))
            return self.fc(x.mean([2, 3]))

    _SHUFFLE_SWAP = {shufflenetv2.InvertedResidual: FusedShuffleInvertedResidual, shufflenetv2.ShuffleNetV2: FusedShuffleNetV2}


try:
    from torchvision.models import vgg
except ImportError:  # without torchvision there is nothing to rewrite
    _VGG_SWAP = {}
else:

    def _vgg_features(features, x):
        """VGG's `features` walked group by group: Conv2d, batch norm and ReLU followed by a max-pool is one
        bn_relu_maxpool site, without one a bn_relu site; every other module (and so every module of a VGG without
        batch norm) is called as a module."""
        mods = list(features)
        i = 0
        while i < len(mods):
            if (i + 2 < len(mods) and type(mods[i]) is nn.Conv2d and isinstance(mods[i + 1], (nn.BatchNorm2d, nn.SyncBatchNorm))
                    and type(mods[i + 2]) is nn.ReLU):
                conv, bn, relu = mods[i:i + 3]
                if i + 3 < len(mods) and type(mods[i + 3]) is nn.MaxPool2d:
                    x = bn_relu_maxpool(bn, relu, mods[i + 3], conv(x))
                    i += 4
                else:
                    x = bn_relu(bn, relu, conv(x))
                    i += 3
            else:
                x = mods[i](x)
                i += 1
        return x

    class FusedVGG(vgg.VGG):
        """VGG whose `features` run group by group: each stage's last Conv2d, batch norm, ReLU and max-pool a
        bn_relu_maxpool site, every other Conv2d, batch norm and ReLU a bn_relu site, anything else its module; avgpool,
        flatten and the classifier run as torchvision runs them.  A `features` that is not an nn.Sequential or has a
        hook of its own, a global hook, and eval with gradients recorded run the parent's forward."""

        def forward(self, x):
            f = self.features
            if (not self.training and torch.is_grad_enabled()) or type(f) is not nn.Sequential or _hooked(f) or _global_hooks():
                return super().forward(x)
            x = self.avgpool(_vgg_features(f, x))
            x = torch.flatten(x, 1)
            return self.classifier(x)

    _VGG_SWAP = {vgg.VGG: FusedVGG}


# Torch sums a tensor of fewer elements than this (2^31 bytes of bf16) in one launch of its reduce kernel, whose order
# the squeeze-excitation kernels restate; a larger one it splits into 32-bit-indexed pieces.
_SE_MAX_NUMEL = 2 ** 30


class _SELink:
    """What a squeeze-excitation site's scale backward hands its pool backward, which runs after the squeeze path's
    backward: s, and dy (channels-last, for the elementwise kernel) or, for a gradient in another layout, eager
    torch's dy * s.  It holds them only from the one backward to the other, and never s's graph: both Functions' ctx
    keep the link, and s's grad_fn leads back to the pool's node through the squeeze path, so a graph-carrying tensor
    on the link would close a cycle through C++ autograd edges that Python's collector cannot free."""

    __slots__ = ("s", "dy", "xgrad")

    def __init__(self):
        self.s = self.dy = self.xgrad = None


def _se_scratch_bytes(x, n, c, hw):
    """The scratch a squeeze-excitation site of x's shape needs on x's device; 0 where the library takes no such site."""
    key = (x.device.index, n, c, hw)
    need = _se_need.get(key)
    if need is None:
        need = _se_need[key] = int(_native_lib().b200c_se_scratch_bytes(n, c, hw))
    return need


def _se_scratch_ptr(x, n, c, hw, stream):
    """The scratch pointer and its size in bytes for a squeeze-excitation site of x's shape on `stream`."""
    ptr = _scratch_ptr(x.device, stream, _se_scratch_bytes(x, n, c, hw), _se_scratch)
    return ptr, _se_scratch[(x.device.index, stream)][0]


def _se_like(t):
    """A tensor like `t` (channels-last [N, C, H, W]) with the strides torch's elementwise ops give s * t or t * s:
    channels-last, except over one row per sample, where every operand is also contiguous and so is the output."""
    n, c, h, w = t.shape
    return torch.empty_like(t) if h * w > 1 else torch.empty((n, c, 1, 1), dtype=t.dtype, device=t.device)


class _SqueezePool(torch.autograd.Function):
    """pooled = x.mean((-1, -2), keepdim=True), with the strides adaptive_avg_pool2d gives it.  The backward writes x's
    whole gradient in one kernel: the mean's (gp / HW) plus the scale's (dy * s, which `link` carries)."""

    @staticmethod
    def forward(ctx, x, link):
        n, c, h, w = x.shape
        pooled = torch.empty((n, c, 1, 1), dtype=x.dtype, device=x.device)
        # adaptive_avg_pool2d restrides the mean of a channels-last input, which it decides from x's strides
        if h * w > 1 or torch._prims_common.suggest_memory_format(x) == torch.channels_last:
            pooled = pooled.as_strided((n, c, 1, 1), (c, 1, c, c))
        stream = _raw_stream(x.device.index)
        scratch, size = _se_scratch_ptr(x, n, c, h * w, stream)
        N.check(_native_lib().b200c_se_pool(x.data_ptr(), pooled.data_ptr(), n, c, h * w, scratch, size, stream))
        ctx.shape, ctx.link = x.shape, link
        ctx.set_materialize_grads(False)
        return pooled

    @staticmethod
    @once_differentiable
    def backward(ctx, gp):
        link, shape = ctx.link, ctx.shape
        dy, s, xgrad = link.dy, link.s, link.xgrad
        link.dy = link.s = link.xgrad = None
        n, c, h, w = shape
        if gp is None or dy is None:
            # eager torch's ops: the scale's gradient (if any) plus the mean's backward, added in place as autograd adds
            if dy is not None:
                xgrad = dy * s
            if gp is None:
                return xgrad, None
            mean_grad = gp.expand(shape) / (h * w)
            return (mean_grad if xgrad is None else xgrad.add_(mean_grad)), None
        gp = gp.reshape(n, c).contiguous()
        s2 = s.reshape(n, c).contiguous()
        dx = _se_like(dy)
        N.check(_native_lib().b200c_se_backward_elemt(dy.data_ptr(), s2.data_ptr(), gp.data_ptr(), dx.data_ptr(), n, c, h * w,
                                                      _raw_stream(dy.device.index)))
        return dx, None


class _SqueezeScale(torch.autograd.Function):
    """y = s * x for s of [N, C, 1, 1].  The backward writes s's gradient (the sum over H, W of dy * x, in torch's
    order) and hands dy to the pool's backward through `link`, which writes x's gradient; where s needs no gradient
    (the pool's backward may then never run) x's gradient is eager torch's dy * s here.

    A gradient that arrives in another layout than channels-last makes eager torch's product and sum run in that layout,
    whose reduction order differs; there the backward runs those torch ops."""

    @staticmethod
    def forward(ctx, s, x, link):
        n, c, h, w = x.shape
        y = _se_like(x)
        s2 = s.reshape(n, c).contiguous()
        N.check(_native_lib().b200c_se_scale(x.data_ptr(), s2.data_ptr(), y.data_ptr(), n, c, h * w, _raw_stream(x.device.index)))
        ctx.link = link
        ctx.save_for_backward(s, x)
        ctx.set_materialize_grads(False)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        if dy is None:
            return None, None, None
        s, x = ctx.saved_tensors
        need_s, need_x = ctx.needs_input_grad[:2]
        link = ctx.link
        ds = dx = None
        if not _activation(dy):
            if need_s:
                ds = (dy * x).sum_to_size(s.shape)
            if need_x:
                if need_s:
                    link.xgrad = (dy * s).detach()
                else:
                    dx = dy * s
            return ds, dx, None
        n, c, h, w = x.shape
        if need_s:
            # sum_to's keepdim sum writes a contiguous [N, C, 1, 1]; over one row it returns the product itself, which is
            # contiguous too (_se_like)
            ds = torch.empty((n, c, 1, 1), dtype=dy.dtype, device=dy.device)
            stream = _raw_stream(x.device.index)
            scratch, size = _se_scratch_ptr(x, n, c, h * w, stream)
            N.check(_native_lib().b200c_se_backward_reduce(dy.data_ptr(), x.data_ptr(), ds.data_ptr(), n, c, h * w, scratch, size,
                                                           stream))
        if need_x:
            if need_s:
                link.dy, link.s = dy.detach(), s.detach()
            else:
                dx = dy * s
        return ds, dx, None


def _se_ok(se, x):
    """Whether squeeze-excitation module `se` can run its pool and scale on the kernels for input x: the conditions of
    the module docstring."""
    if not _activation(x) or x.numel() == 0 or x.numel() >= _SE_MAX_NUMEL:
        return False
    n, c, h, w = x.shape
    if c == 1 and h * w > 1:   # torch reduces one channel along its fastest dimension, in another order
        return False
    pool = se.avgpool
    if type(pool) is not nn.AdaptiveAvgPool2d or pool.output_size not in (1, (1, 1)) or _skips_hooks(pool):
        return False
    return _se_scratch_bytes(x, n, c, h * w) > 0


try:
    from torchvision.ops.misc import SqueezeExcitation
except ImportError:  # without torchvision there is nothing to rewrite
    SqueezeExcitation = None
else:

    class FusedSqueezeExcitation(SqueezeExcitation):
        """torchvision's SqueezeExcitation whose average pool and scale run on the squeeze-excitation kernels: the pool,
        then fc1, activation, fc2 and scale_activation called as modules, then the scale.  Both writes and both
        gradients of x (the scale's and the mean's) have eager torch's bits; the backward reads x and dy twice and
        writes dx once.  Runs the parent's forward where the kernels do not apply (the module docstring), and torch's
        `s * x` where the squeeze path returns anything but a bf16 [N, C, 1, 1] on x's device."""

        def forward(self, input):
            if not _se_ok(self, input):
                return super().forward(input)
            link = _SELink()
            s = self.scale_activation(self.fc2(self.activation(self.fc1(_SqueezePool.apply(input, link)))))
            n, c = input.shape[:2]
            if not (isinstance(s, torch.Tensor) and s.dtype == torch.bfloat16 and s.device == input.device
                    and s.shape == (n, c, 1, 1)):
                return s * input
            return _SqueezeScale.apply(s, input, link)


def fuse_model(model):
    """Rewrite `model` in place: `fuse_resnet`, and every module whose class is exactly torchvision's
    Conv2dNormActivation and whose last module is an nn.ReLU6, SiLU or Hardswish (MobileNetV2 / V3, EfficientNet)
    becomes a FusedConv2dNormActivation.  Every module whose class is exactly torchvision's MobileNetV2 or MobileNetV3
    InvertedResidual or EfficientNet's MBConv gets the fused subclass, whose projection batch norm (with the stochastic
    depth and residual add after it) runs as one bn_res site, and every SqueezeExcitation (exactly that class) inside such
an MBConv or MobileNetV3 block becomes a FusedSqueezeExcitation.  Every module whose class is exactly torchvision's
    DenseNet, _DenseBlock or _DenseLayer gets the fused subclass, whose concatenating batch norms run as concatenation
    sites (`bn_relu_cat`).  Every module whose class is exactly torchvision's Inception v3 or GoogLeNet BasicConv2d,
    InceptionA to InceptionE or GoogLeNet's Inception gets the fused subclass: BasicConv2d's batch norm and ReLU run as
    a bn_relu site, and each Inception module's branches write their last batch norm and ReLU into their channels of the
    module's output (`bn_relu_concat`).  Every module whose class is exactly torchvision's ShuffleNetV2 or its
    InvertedResidual gets the fused subclass: the stem is one bn_relu_maxpool site, conv5 a bn_relu site, and each
    block's branches run module by module into one block-end site that writes the shuffled output directly
    (`bn_relu_shuffle`).  Every module whose class is exactly torchvision's VGG gets the fused subclass: each stage's
    last batch norm, ReLU and 2 x 2 max-pool is one bn_relu_maxpool site and every other batch norm and ReLU a bn_relu
    site (a VGG without batch norm runs torchvision's ops).  Parameters, buffers, state_dict keys, hooks and the
    object itself are unchanged, and a second call changes nothing.  Every fused site has eager torch's bits, in
    training and in eval (see `fuse_resnet` for inference).

    RegNet's squeeze-excitation and SqueezeExcitation modules outside those blocks keep torchvision's class.  Blocks
    ending in nn.ReLU (MobileNetV3, RegNet) keep torchvision's forward: bn_act would run them on bn_relu's sites,
    but a regnet_y_400mf training step with them fused took about 11 ms more host time than the untouched model (DESIGN.md
    section 10), more than the kernel time they save."""
    fuse_resnet(model)
    if Conv2dNormActivation is not None:
        for mod in model.modules():
            if type(mod) is Conv2dNormActivation and len(mod) == 3 and type(mod[2]) in _ACT_CODES:
                mod.__class__ = FusedConv2dNormActivation
    swap = {**_RES_SWAP, **_DENSE_SWAP, **_SLICE_SWAP, **_SHUFFLE_SWAP, **_VGG_SWAP}
    for mod in model.modules():
        cls = swap.get(type(mod))
        if cls is not None:
            mod.__class__ = cls
    if SqueezeExcitation is not None and _RES_SWAP:
        for mod in model.modules():
            if type(mod) in (FusedMBConv, FusedInvertedResidualV3):
                for sub in mod.modules():
                    if type(sub) is SqueezeExcitation:
                        sub.__class__ = FusedSqueezeExcitation
    return model


def fuse_resnet(model):
    """Rewrite `model` in place: every module whose class is exactly torchvision's ResNet, Bottleneck or BasicBlock
    gets the fused subclass.  Parameters, buffers, state_dict keys, hooks and the object itself are unchanged.

    This is also the entry point for inference: after `model.eval()`, a forward under `torch.inference_mode()` or
    `torch.no_grad()` on bf16 channels-last input (autocast with fp32 parameters, or a model cast to bf16) runs every
    batch norm of the model, with the ReLU, residual add and stem max-pool after it, as one native launch per site,
    bit-identical to the untouched model."""
    for mod in model.modules():
        cls = _SWAP.get(type(mod))
        if cls is not None:
            mod.__class__ = cls
    return model
