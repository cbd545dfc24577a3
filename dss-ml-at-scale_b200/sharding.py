"""Multi-GPU: hash-shard the groups, fit with zero communication, one all-gather at the end.

The reference spreads groups with ``repartition(n_tasks, "Product", "SKU")`` -- a hash
shuffle of the key columns -- and then runs one task per group
(group_apply/02_Fine_Grained_Demand_Forecasting.py:520-528).  Groups are independent, so
the H100 analogue is: ``owner = hash(key) mod world_size`` at pack time, every rank fits
its own series (no data-path collective), and exactly one ``all_gather`` of the
``[per_rank, n_pred]`` float32 forecast table over NCCL (NVLink / NVSwitch) gives every
rank the whole table.  One process per GPU; ``torch.distributed`` is the plumbing.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


def stable_hash64(key_frame) -> np.ndarray:
    """Deterministic 64-bit hash of the key columns (same on every rank / every run)."""
    import pandas as pd

    return pd.util.hash_pandas_object(key_frame, index=False).to_numpy(dtype=np.uint64)


def owner_of_keys(key_frame, world: int) -> np.ndarray:
    """``hash(key) mod world`` -- the analogue of ``repartition(n, keys)`` (02:525)."""
    return (stable_hash64(key_frame) % np.uint64(world)).astype(np.int64)


def owner_of_rows(n: int, world: int) -> np.ndarray:
    """Packed benchmarks have no keys: contiguous equal blocks of ceil(n/world) rows."""
    per = -(-n // world)
    return np.minimum(np.arange(n, dtype=np.int64) // per, world - 1)


@dataclass
class ShardPlan:
    world: int
    rank: int
    owner: np.ndarray        # [n] rank that fits series i
    per: int                 # rows of every rank's padded table (max shard size)
    local_rows: np.ndarray   # indices of this rank's series, ascending
    slot: np.ndarray         # [n] position of series i inside its owner's padded table

    @staticmethod
    def build(owner: np.ndarray, world: int, rank: int) -> "ShardPlan":
        owner = np.asarray(owner, dtype=np.int64)
        counts = np.bincount(owner, minlength=world)
        per = int(max(int(counts.max()) if owner.size else 0, 1))
        order = np.argsort(owner, kind="stable")
        starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
        slot = np.empty(owner.size, dtype=np.int64)
        slot[order] = np.arange(owner.size) - starts[owner[order]]
        return ShardPlan(world, rank, owner, per, np.flatnonzero(owner == rank), slot)

    def gather_index(self) -> np.ndarray:
        """Row of the gathered ``[world*per, n_pred]`` table that holds series i."""
        return self.owner * self.per + self.slot


def all_gather_table(local, plan: ShardPlan, group=None):
    """``local`` [per, n_pred] (rows >= this rank's shard size are padding) ->
    ``[n, n_pred]`` in the original series order on every rank.  One collective."""
    import torch
    import torch.distributed as dist

    gathered = torch.empty((plan.world * plan.per, local.shape[1]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(gathered, local.contiguous(), group=group)
    idx = torch.as_tensor(plan.gather_index(), device=local.device)
    return gathered.index_select(0, idx)


def all_gather_inplace(table, plan: ShardPlan, group=None):
    """In-place flavour for packed data: ``table`` is the full ``[world*per, n_pred]`` buffer and
    this rank's kernel already wrote rows ``[rank*per, (rank+1)*per)`` -- no staging copy."""
    import torch.distributed as dist

    mine = table[plan.rank * plan.per:(plan.rank + 1) * plan.per]
    dist.all_gather_into_tensor(table, mine, group=group)
    return table


def forecast_packed_sharded(y_local, plan: ShardPlan, engine, pred_start: int, n_pred: int, group=None):
    """Fit this rank's packed series ``y_local`` [len(plan.local_rows), T] (torch CUDA tensor or NumPy)
    and return the whole ``[n, n_pred]`` forecast table (torch tensor) on every rank."""
    import torch

    n_local = plan.local_rows.size
    is_t = type(y_local).__module__.startswith("torch")
    if is_t:
        local = torch.zeros((plan.per, n_pred), dtype=torch.float32, device=y_local.device)
        if n_local:
            engine.fit_forecast(y_local, pred_start, n_pred, out=local[:n_local])
    else:
        buf = np.zeros((plan.per, n_pred), dtype=np.float32)
        if n_local:
            engine.fit_forecast(y_local, pred_start, n_pred, out=buf[:n_local])
        local = torch.from_numpy(buf)
    return all_gather_table(local, plan, group)


class SymmetricTable:
    """The gathered forecast table ``[world * per, n_pred]`` in NVLink symmetric memory
    (``torch.distributed._symmetric_memory``): every rank owns a full copy, peers' copies are mapped into
    this process and -- when the fabric supports NVLS -- one multicast address reaches all of them.
    ``ForecastEngine.fit_forecast_bcast`` then writes each forecast row into every copy from the fit
    kernel's epilogue, so no separate all-gather runs; ``barrier()`` orders the reads."""

    def __init__(self, per: int, n_pred: int, device, group=None, mode: str = "p2p"):
        """mode: "p2p" (bulk stores to every peer copy, default), "multicast" (multimem.st to the NVLS
        address) or "multicast-bulk" (bulk stores to the NVLS address)."""
        import torch
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem

        group = group or dist.group.WORLD
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.per, self.n_pred = per, n_pred
        self.table = symm_mem.empty((self.world * per, n_pred), dtype=torch.float32, device=device)
        self.table.zero_()
        self.handle = symm_mem.rendezvous(self.table, group.group_name if hasattr(group, "group_name") else group)
        slice_bytes = self.rank * per * n_pred * 4
        mc = int(getattr(self.handle, "multicast_ptr", 0) or 0)
        if mode != "p2p" and not mc:
            raise RuntimeError("no NVLS multicast address available for this group")
        self.multimem = {"p2p": 0, "multicast": 1, "multicast-bulk": 2}[mode]
        if self.multimem:
            self.out_ptrs = [mc + slice_bytes]
        else:
            # own copy first, then the peers' (P2P stores) starting at rank+1: no two ranks walk the peers in the same
            # order, so no GPU's NVLink ingress is every sender's first target (the kernel additionally starts
            # each tile at a different peer)
            order = [self.rank] + [(self.rank + k) % self.world for k in range(1, self.world)]
            self.out_ptrs = [int(self.handle.buffer_ptrs[r]) + slice_bytes for r in order]

    def barrier(self):
        self.handle.barrier()

    def fit_into(self, engine, y_local, pred_start: int, n_pred: int, status=None):
        """Fit this rank's rows and broadcast their forecasts into every rank's table copy."""
        engine.fit_forecast_bcast(y_local, pred_start, n_pred, self.out_ptrs, self.n_pred, self.multimem, status=status)


def forecast_groups_sharded(pdf, *, keys=("Product", "SKU"), group=None, gather: bool = True, engine=None, **kw):
    """DataFrame-level analogue of the reference's distributed fan-out (02:520-528), one process per GPU:
    ``owner = hash(key) mod world`` (the ``repartition(n_tasks, "Product", "SKU")`` shuffle), every rank runs
    ``forecast_groups`` on the groups it owns -- no communication during the fit -- and, with ``gather=True``,
    every rank ends up with the whole ``tuning_schema`` frame (groups in key order).  ``pdf`` must hold all rows
    of the groups this rank owns (e.g. the same frame on every rank, or a frame pre-partitioned by the same hash).
    For packed data use ``ShardPlan`` + ``forecast_packed_sharded`` / ``SymmetricTable`` (numeric table only)."""
    import pandas as pd
    import torch.distributed as dist

    from .frames import forecast_groups

    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    keys = list(keys)
    owner = owner_of_keys(pdf[keys], world) if len(pdf) else np.zeros(0, dtype=np.int64)
    local = forecast_groups(pdf[owner == rank], keys=keys, engine=engine, **kw)
    if not gather or world == 1:
        return local
    parts = [None] * world
    dist.all_gather_object(parts, local, group=group)
    out = pd.concat([p for p in parts if len(p)], ignore_index=True) if any(len(p) for p in parts) else local
    date_col = kw.get("date_col", "Date")
    return out.sort_values(keys + [date_col], kind="stable", ignore_index=True)
