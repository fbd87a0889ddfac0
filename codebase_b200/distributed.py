"""Data-parallel training over the processes `torchrun` starts (weak scaling, DESIGN.md section 5).

    torchrun --nproc-per-node 2 -m codebase_b200.run +algorithm=idqn env.name="lbforaging:Foraging-8x8-2p-3f-v3" env.time_limit=25

Rank r owns env.parallel_envs envs with global ids [r * P, (r + 1) * P) and its own replay ring or on-policy batch.  One update sums the
un-normalised gradient sums, loss numerators and filled counts of all ranks; every rank then divides by the global filled count, clips by the
global norm and applies the same optimiser step, so replicated parameters stay bit-identical.  Without torchrun's variables, or with
WORLD_SIZE=1, nothing here starts a process group and every code path is the single-process one.

Collectives: nccl on the device buffers when every rank has its own device (the ranks' device UUIDs differ), gloo on host copies of them
otherwise (several ranks sharing one device).
"""
from __future__ import annotations

import os

import torch

MAX_RANKS = 8   # kMaxRanks (csrc/learner.cuh): the largest world of the in-kernel gradient exchange


class DataParallel:
    """This process's place in the data-parallel group; the single-process instance (world 1) makes every collective the identity."""

    def __init__(self, rank=0, world=1, local_rank=0, local_world=1, backend=None, device_index=None):
        self.rank, self.world, self.local_rank, self.local_world = int(rank), int(world), int(local_rank), int(local_world)
        self.backend, self.device_index = backend, device_index

    @property
    def active(self) -> bool:
        return self.world > 1

    @property
    def is_main(self) -> bool:
        return self.rank == 0

    @property
    def own_device(self) -> bool:
        """Every rank has a device of its own (the in-kernel peer exchange needs co-resident peers on distinct devices)."""
        return self.backend == "nccl"

    def _coll_device(self):
        return torch.device("cuda", self.device_index) if self.backend == "nccl" else torch.device("cpu")

    def sum_int(self, x: int) -> int:
        """The sum of an integer over all ranks: one int64 all-reduce (identity on one rank)."""
        if not self.active:
            return int(x)
        import torch.distributed as dist

        t = torch.tensor([int(x)], dtype=torch.int64, device=self._coll_device())
        dist.all_reduce(t)
        return int(t.item())

    def all_reduce_(self, tensors):
        """Sum each tensor over all ranks, in place.  Every rank ends with the same bits."""
        if not self.active:
            return
        import torch.distributed as dist

        if self.backend == "nccl":
            for t in tensors:
                dist.all_reduce(t)
            return
        flat = torch.cat([t.detach().reshape(-1).cpu() for t in tensors])   # gloo: one exchange of host copies
        dist.all_reduce(flat)
        o = 0
        for t in tensors:
            t.copy_(flat[o:o + t.numel()].view_as(t))
            o += t.numel()

    def broadcast_(self, tensors, src=0):
        """Overwrite each tensor with rank `src`'s copy."""
        if not self.active:
            return
        import torch.distributed as dist

        for t in tensors:
            if self.backend == "nccl":
                dist.broadcast(t, src)
            else:
                h = t.detach().cpu()
                dist.broadcast(h, src)
                t.copy_(h)

    def broadcast_object(self, obj, src=0):
        if not self.active:
            return obj
        import torch.distributed as dist

        box = [obj]
        dist.broadcast_object_list(box, src)
        return box[0]

    def gather_objects(self, obj) -> list:
        """[obj of rank 0, obj of rank 1, ...] on every rank."""
        if not self.active:
            return [obj]
        import torch.distributed as dist

        out = [None] * self.world
        dist.all_gather_object(out, obj)
        return out

    def sync_learner(self, model):
        """Start every rank from rank 0's parameters and targets (and the QMIX mixer's), so that equal starts do not depend on equal RNG streams."""
        if not self.active:
            return
        bufs = [model.theta, model.theta_tgt]
        if getattr(model, "mix", None) is not None:
            bufs += [model.mix, model.mix_tgt]
        self.broadcast_(bufs)
        if hasattr(model, "params_changed"):
            model.params_changed()


_current = DataParallel()


def current() -> DataParallel:
    """The group set up by `init` (the single-process instance before, or without torchrun)."""
    return _current


def from_environ(environ=None):
    """(rank, world, local_rank, local_world) from torchrun's variables; (0, 1, 0, 1) without them."""
    env = os.environ if environ is None else environ
    world = int(env.get("WORLD_SIZE", "1"))
    rank, local = int(env.get("RANK", "0")), int(env.get("LOCAL_RANK", "0"))
    local_world = int(env.get("LOCAL_WORLD_SIZE", str(world)))
    return rank, world, local, local_world


def check_supported(cfg, world: int, local_world: int):
    """What data-parallel training does not cover yet; raised before any native call."""
    if world <= 1:
        return
    if world > MAX_RANKS:
        raise NotImplementedError(f"WORLD_SIZE={world}: data-parallel training runs on at most {MAX_RANKS} ranks")
    if local_world != world:
        raise NotImplementedError(f"WORLD_SIZE={world} with LOCAL_WORLD_SIZE={local_world}: data-parallel training runs on one node")
    if bool(cfg.algorithm.get("standardise_returns", False)):
        raise NotImplementedError("algorithm.standardise_returns=True with WORLD_SIZE > 1: each rank's return statistics would see different returns and "
                                  "the replicas would diverge (the statistics are not exchanged)")


def choose_backend(device_uuids) -> str:
    """nccl when every rank has a device of its own (the ranks' device UUIDs are all distinct), gloo when ranks share devices (or have none).
    UUIDs rather than device counts: a launcher that shows each process only its own GPU gives every rank device_count() == 1."""
    return "nccl" if all(u is not None for u in device_uuids) and len(set(device_uuids)) == len(device_uuids) else "gloo"


def shard(rank: int, parallel_envs: int) -> int:
    """The first global env id of rank `rank` (its envs are [rank * P, (rank + 1) * P))."""
    return int(rank) * int(parallel_envs)


def init(cfg, environ=None) -> DataParallel:
    """Read torchrun's variables, refuse what is not supported, select the device (LOCAL_RANK % device_count) and start the process group."""
    global _current
    rank, world, local, local_world = from_environ(environ)
    check_supported(cfg, world, local_world)
    if world <= 1:
        _current = DataParallel()
        return _current
    import torch.distributed as dist

    n_dev = torch.cuda.device_count()
    dev = local % n_dev if n_dev else None
    if dev is not None:   # gloo for host objects and host copies, nccl (created on first use) for device tensors
        torch.cuda.set_device(dev)
        dist.init_process_group("cpu:gloo,cuda:nccl")
    else:
        dist.init_process_group("gloo")
    uuids = [None] * world
    dist.all_gather_object(uuids, str(torch.cuda.get_device_properties(dev).uuid) if dev is not None else None)
    _current = DataParallel(rank, world, local, local_world, choose_backend(uuids), dev)
    return _current


def finish():
    """Leave the process group (no-op on one rank)."""
    global _current
    if _current.active:
        import torch.distributed as dist

        dist.destroy_process_group()
    _current = DataParallel()
