"""Data-parallel learner over the GPUs of one box (SURVEY.md section 8e; BASELINE config 5).

The reference has a single learner process and no collective at all (its "distributed" layer is Redis over
TCP).  Here each rank owns one GPU, one replay shard and one replica of the networks; the learner step is
independent per transition up to the gradient reduction, so the only data-path collective is ONE all-reduce
(NCCL over NVLink/NVSwitch) of the flat fp32 gradient arena per step, followed by an identical Adam step on
every rank (grad_scale = 1/world_size makes it the mean over the global batch, like `(weights*loss).mean()`
over B*world transitions).  Equivalence to a single-GPU learner on the concatenated batch requires the SAME
noisy-layer epsilons on every rank for each of the three resets per step -- the ranks share the Philox seed and
advance the same counters -- while the quantile fractions tau are per-row and use a per-rank stream.
"""
import os

import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """torchrun-style init (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_*).  Returns (rank, world, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def shard_batch(global_batch, world):
    """Per-rank minibatch of a strong-scaling run (global batch fixed)."""
    if global_batch % world:
        raise ValueError("global batch must divide by the number of ranks")
    return global_batch // world


def broadcast_seed(seed, group=None, device="cpu"):
    t = torch.tensor([seed], dtype=torch.int64, device=device)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.broadcast(t, src=0, group=group)
    return int(t.item())


def make_data_parallel(learner, group=None):
    """Turn a Learner into one replica of a data-parallel learner: parameters, epsilons and noise seeds are
    broadcast from rank 0; gradients are summed across ranks before Adam; tau streams are made rank-private."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return learner
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    dev = learner.online_net._flat.device
    for net in (learner.online_net, learner.target_net):
        dist.broadcast(net._flat, src=0, group=group)
        dist.broadcast(net._eps_flat, src=0, group=group)
        net._rng_seed = broadcast_seed(net._rng_seed, group, dev)
        net._tau_stream_offset = rank << 40
        for _, m in net.noisy_layers():
            m._noise_calls = 0
        if net._flat.is_cuda:
            net.compose_weights()
    if getattr(learner, "fraction_net", None) is not None:        # FQF: the fraction proposal's own arena
        dist.broadcast(learner.fraction_net._flat, src=0, group=group)
        learner.fraction_optimiser.grad_scale = 1.0 / world
    if getattr(learner, "curl_net", None) is not None:             # CURL: the projection and the momentum encoder
        for t in (learner.curl_net._flat, learner.momentum_net._flat, learner.momentum_projection):
            dist.broadcast(t, src=0, group=group)
        learner.curl_optimiser.grad_scale = 1.0 / world
    if getattr(learner, "spr_net", None) is not None:              # SPR: projection, transition model, predictor
        dist.broadcast(learner.spr_net._flat, src=0, group=group)
        learner.spr_optimiser.grad_scale = 1.0 / world
    learner.process_group = group if group is not None else dist.group.WORLD
    learner.optimiser.grad_scale = 1.0 / world
    return learner


def publish_parameters(agent, src=0, group=None):
    """Ape-X parameter publication over the collective fabric: the learner rank broadcasts its flat parameter arena
    (26.9 MB; the epsilon buffers are not sent -- actors resample noise, launch_actor.py:76-77) and every other rank
    (actor GPUs) receives it.  Replaces Learner.save_to_redis / Actor.load_weight_from_redis (learner.py:28-36,
    actor.py:36-39), which ship a torch.save blob through Redis every weight_synchro_frequency steps."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    net = agent.online_net
    dist.broadcast(net._flat, src=src, group=group)
    if getattr(agent, "fraction_net", None) is not None:          # FQF: actors act on the learner's fractions
        dist.broadcast(agent.fraction_net._flat, src=src, group=group)
    if dist.get_rank(group) != src and net._flat.is_cuda:
        net.compose_weights()


def allreduce_sum(value, device):
    t = torch.tensor([value], dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


def allreduce_max(value, device):
    t = torch.tensor([value], dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
