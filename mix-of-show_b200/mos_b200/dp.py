"""Data-parallel plumbing of ED-LoRA training (SURVEY.md §8e): one process per GPU, the image batch is sharded across
ranks, weights are replicated, and the ONLY data-path collective is a single all-reduce per optimiser step on one
flat fp32 buffer [concept rows | text-encoder LoRA | UNet LoRA | 2 logged scalars] (4.47 MB for SD1.5), replacing the
156 MB the reference's DDP moves (train_edlora.py:70,128; util.py:203-229).  torch.distributed is the transport
(NCCL over NVLink on the GPU box, gloo in the CPU tests); the arithmetic after it is mos_flat_adamw_step.
Gradient fusion shards by layer instead (gradient_fusion.fusion_plan): every rank solves its own layers and the solved
weights are broadcast by their owners (all_ranks_ok, broadcast_owned).
"""
import math

import torch
import torch.distributed as dist


class FlatTrainState:
    """Flat parameter / gradient / Adam-moment buffers with the three learning-rate groups of train_edlora.py:57.  A group
    that does not train has zero length.  `const_rows`: when the embedding group does not train, a state of its own
    over the (constant) concept rows, so that optimizer_step still reduces their Norm_mean every step
    (train_edlora.py:138-140)."""

    def __init__(self, n_emb_rows, emb_dim, n_text_lora, n_unet_lora, lrs=(1e-3, 1e-5, 1e-4), device='cpu'):
        self.emb_rows, self.emb_dim = n_emb_rows, emb_dim
        n0 = n_emb_rows * emb_dim
        self.group_end = (n0, n0 + n_text_lora, n0 + n_text_lora + n_unet_lora)
        self.lrs = tuple(lrs)
        n = self.group_end[2]
        self.params = torch.zeros(n, device=device)
        self.grads = torch.zeros(n + 2, device=device)        # + [loss, Norm_mean] riding on the same collective
        self.exp_avg = torch.zeros(n, device=device)
        self.exp_avg_sq = torch.zeros(n, device=device)
        self.step = 0
        self.const_rows = None

    @property
    def group_sizes(self):
        return (self.group_end[0], self.group_end[1] - self.group_end[0], self.group_end[2] - self.group_end[1])

    @property
    def has_rows(self):
        """whether optimizer_step can report Norm_mean of the concept rows"""
        return self.emb_rows > 0 or self.const_rows is not None

    def set_const_rows(self, rows):
        """rows fp32 [R, C]: the concept rows of an untrained embedding group (see the class docstring)"""
        R, C = rows.shape
        c = FlatTrainState(R, C, 0, 0, lrs=(0.0, 0.0, 0.0), device=self.params.device)
        c.params.copy_(rows.reshape(-1))
        self.const_rows = c

    @property
    def n(self):
        return self.group_end[2]


def shard_batch(global_batch, rank, world):
    """Indices of the samples rank `rank` processes (contiguous shards, remainder spread over the first ranks)."""
    base, rem = divmod(global_batch, world)
    start = rank * base + min(rank, rem)
    return list(range(start, start + base + (1 if rank < rem else 0)))


def allreduce_flat(state, loss_value=0.0, norm_mean=0.0, group=None):
    """The one collective of a training step: SUM over ranks of [grads | loss | Norm_mean]; returns
    (grad_scale, mean loss, mean Norm_mean) with DDP's mean semantics (divide by world size)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    state.grads[state.n] = loss_value
    state.grads[state.n + 1] = norm_mean
    if world > 1:
        dist.all_reduce(state.grads, op=dist.ReduceOp.SUM, group=group)
    logs = state.grads[state.n:].tolist()
    return 1.0 / world, logs[0] / world, logs[1] / world


def allreduce_flat_device(state, loss_dev=None, group=None):
    """Same single collective without any host synchronisation: the loss rides on the wire as a device scalar and is
    read later from state.grads[state.n] (divide by the world size).  Returns grad_scale = 1 / world."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if loss_dev is not None:
        state.grads[state.n:state.n + 1].copy_(loss_dev.reshape(1))
    if world > 1:
        dist.all_reduce(state.grads, op=dist.ReduceOp.SUM, group=group)
    return 1.0 / world


def collective_device(device):
    """device the tensors of a collective live on: `device` under NCCL, host memory under gloo (which the ranks use when
    they share one GPU)"""
    return torch.device('cpu') if dist.get_backend() == 'gloo' else torch.device(device)


def all_ranks_ok(ok, device):
    """MIN-all-reduce of a success flag before a result exchange: a rank whose work raised says so here, so every rank
    learns of the failure instead of waiting in a broadcast that rank never joins."""
    flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=collective_device(device))
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    return bool(flag.item())


def broadcast_owned(owned, plan, shapes, device):
    """Exchange of a sharded gradient-fusion stage: plan[r] lists the weights rank r solved (gradient_fusion.fusion_plan),
    `owned` holds this rank's as fp32 tensors on `device`.  Each owner broadcasts its weights in plan order as ONE flat
    buffer, so a stage costs `world` broadcasts whatever its layer count.  -> {name: fp32 tensor of shapes[name]} for every
    weight of the plan: this rank's own tensors as given, the others' on collective_device(device) (host memory under
    gloo, where the caller wants them next)."""
    rank = dist.get_rank()
    wire = collective_device(device)
    out = {}
    for r, names in enumerate(plan):
        if not names:
            continue
        sizes = [math.prod(shapes[n]) for n in names]
        if r == rank:
            buf = torch.cat([owned[n].reshape(-1) for n in names]).to(wire, torch.float32)
        else:
            buf = torch.empty(sum(sizes), dtype=torch.float32, device=wire)
        dist.broadcast(buf, src=r)
        if r == rank:
            out.update((n, owned[n]) for n in names)
            continue
        for n, part in zip(names, buf.split(sizes)):
            out[n] = part.view(shapes[n])
    return out


def optimizer_step(state, grad_scale, norm_out=None):
    """AdamW on the flat state (CUDA only: there is no CPU fallback for the arithmetic)."""
    from . import ops
    if not state.params.is_cuda:
        raise RuntimeError('optimizer_step needs the flat state on a CUDA device (no CPU fallback)')
    state.step += 1
    ops.flat_adamw_step(state.params, state.grads, state.exp_avg, state.exp_avg_sq, state.group_end, state.lrs,
                        step=state.step, grad_scale=grad_scale, emb_rows=state.emb_rows, emb_dim=state.emb_dim,
                        norm_mean_out=norm_out)
    c = state.const_rows
    if norm_out is not None and state.emb_rows == 0 and c is not None:
        # Norm_mean of constant rows through the same reduction: an AdamW step at learning rate 0 on zero gradients
        # leaves the rows (and the zero moments) bit-identical: p (1 - 0 wd) - 0 m / (sqrt(v) + eps) = p
        ops.flat_adamw_step(c.params, c.grads, c.exp_avg, c.exp_avg_sq, c.group_end, c.lrs, step=1,
                            emb_rows=c.emb_rows, emb_dim=c.emb_dim, norm_mean_out=norm_out)
