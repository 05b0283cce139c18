"""Multi-GPU plumbing for the hook-chain path: payloads are independent units, so a batch is
partitioned across ranks (size-balanced) and every rank scans its own shard; the ONLY exchange is
one all-gather of the per-unit verdict bitmaps (24-ish bytes per payload; payload bytes never cross
NVLink).  torch.distributed is plumbing here: NCCL on the GPUs, gloo in the CPU tests.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np

from ._native import CF_STAGE_MASK


def partition_units(sizes: Sequence[int], world: int) -> List[List[int]]:
    """Greedy size-balanced assignment (longest first) of unit indices to ranks; each rank's list is
    returned in ascending unit order so verdicts can be scattered back deterministically."""
    order = sorted(range(len(sizes)), key=lambda i: (-sizes[i], i))
    loads = [0] * world
    parts: List[List[int]] = [[] for _ in range(world)]
    for i in order:
        r = min(range(world), key=lambda k: (loads[k], k))
        parts[r].append(i)
        loads[r] += sizes[i] + 1
    for p in parts:
        p.sort()
    return parts


def gather_verdicts(local: "np.ndarray | object", counts: Sequence[int], words: int, group=None):
    """All-gather variable-length verdict arrays (AllGatherv emulated by padding to the largest shard,
    one collective).  `local` is a torch tensor (int64, n_local * words) on the rank's device.
    Returns the list of per-rank tensors trimmed to their true lengths."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    mx = max(counts) * words
    buf = torch.zeros(mx, dtype=torch.int64, device=local.device)
    buf[: local.numel()] = local
    out = torch.empty(world * mx, dtype=torch.int64, device=local.device)
    dist.all_gather_into_tensor(out, buf, group=group)
    return [out[r * mx: r * mx + counts[r] * words] for r in range(world)]


def scatter_back(parts: List[List[int]], gathered, words: int, n_units: int) -> np.ndarray:
    """Global verdict array (n_units * words, uint64) from the per-rank gathered tensors."""
    full = np.zeros(n_units * words, dtype=np.uint64)
    for idxs, t in zip(parts, gathered):
        a = t.cpu().numpy().view(np.uint64).reshape(-1, words)
        for j, u in enumerate(idxs):
            full[u * words:(u + 1) * words] = a[j]
    return full


class ShardedChain:
    """The hook chain over a batch that is partitioned across the ranks of a torch.distributed group (one process per GPU):
    SURVEY.md §8(b) `cf_run_batch_sharded`.  Every rank runs the fused chain (engine.run_batch: ONE upload, scan + regex_filter
    rewriting + TOON on the resident shard) over ITS units only — payload bytes never cross NVLink — and the per-unit 24-byte
    verdict records are exchanged with ONE all-gather (padded to the largest shard: NCCL has no AllGatherv), so that every rank
    (and the host thread that owns the event loop) sees the verdict of every payload.  Rewritten / re-encoded texts stay with
    their owner rank, as in the design contract.  On NCCL the shard runs through cf_run_enqueue (engine.Run) on the current
    stream and the collective takes the verdict records straight from device memory on that stream; the host copies come after it.

        sc = ShardedChain(prog)                       # after torch.distributed.init_process_group(...)
        parts = sc.partition([len(u) for u in units]) # identical on every rank (deterministic, size-balanced, longest first)
        verdicts, mine, out, out_offs = sc.run(units, parts, stage_mask, unit_stages)
        # verdicts: engine.VERDICT_DTYPE[n_units] in GLOBAL unit order; mine = this rank's unit indices; out/out_offs = their texts
    """

    def __init__(self, prog, device: int | None = None, group=None):
        import torch
        import torch.distributed as dist

        from . import engine

        self.engine = engine
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.backend = dist.get_backend(group)
        self.device = device if device is not None else (torch.cuda.current_device() if torch.cuda.is_available() else None)
        self.prog = prog
        self.ctx = None
        self.batch = None
        self.run_dev = None

    def partition(self, sizes: Sequence[int]) -> List[List[int]]:
        return partition_units(sizes, self.world)

    def _local(self, units, stage_mask: int, unit_stages, toon_flags: int, mask_max_depth: int = 10):
        """This rank's shard through the fused chain (GPU).  Overridable: the gloo CPU test substitutes the oracle here."""
        engine = self.engine
        if self.ctx is None:
            self.ctx = engine.Context.get(self.device or 0)
            if self.prog is not None and self.prog.h is None:
                self.prog.compile(self.ctx)
        enc = [engine.encode_unit(u) for u in units]
        stream, offs = engine.pack_units(enc)
        b = self.batch
        if b is None or len(stream) > b.max_bytes or len(enc) > b.max_units:
            self.batch = b = engine.Batch(self.ctx, max(len(stream) * 2, 1 << 20), max(len(enc) * 2, 1024))
        v, out, oo, _ = engine.run_batch(self.prog, b, stream, offs, stage_mask, unit_stages, toon_flags, mask_max_depth)
        return v, out, oo

    def _enqueue_device(self, units, stage_mask: int, unit_stages, toon_flags: int, words: int, mask_max_depth: int = 10):
        """NCCL: this rank's shard through cf_run_enqueue on the current stream, verdict records left in device memory (int64 words)
        for the collective.  Returns (records, finish), finish() -> (out, out_offsets) on the host once the chain is done."""
        import torch

        engine = self.engine
        if self.ctx is None:
            self.ctx = engine.Context.get(self.device or 0)
            if self.prog is not None and self.prog.h is None:
                self.prog.compile(self.ctx)
        enc = [engine.encode_unit(u) for u in units]
        stream, offs = engine.pack_units(enc)
        n = len(enc)
        b = self.batch
        if b is None or len(stream) > b.max_bytes or n > b.max_units or self.run_dev is None:
            self.batch = b = engine.Batch(self.ctx, max(len(stream) * 2, 1 << 20), max(n * 2, 1024))
            self.run_dev = engine.Run(self.ctx, b.max_units, b.max_bytes)
        dev = torch.device("cuda", self.device or 0)
        cs = torch.cuda.current_stream(dev)
        b.upload(stream, offs, cuda_stream=cs.cuda_stream)
        d_us = None if unit_stages is None else torch.from_numpy(np.ascontiguousarray(unit_stages, dtype=np.uint8)).to(dev, non_blocking=False)
        d_v = torch.empty(n * words, dtype=torch.int64, device=dev)
        d_oo = torch.empty(n + 1, dtype=torch.int64, device=dev)
        state = {"out": torch.empty(max(len(stream), 16), dtype=torch.uint8, device=dev)}

        def enqueue():
            self.run_dev.enqueue(self.prog, b, stage_mask, d_us, toon_flags, d_v, d_oo, state["out"], stream=cs, mask_max_depth=mask_max_depth)

        def finish():
            need = self.run_dev.finish()
            if need:                                      # rewritten or masked texts outgrew the input's size: once more with the room they need
                state["out"] = torch.empty(need, dtype=torch.uint8, device=dev)
                enqueue()
                self.run_dev.finish()
            oo = d_oo.cpu().numpy().view(np.uint64)
            return state["out"][: int(oo[-1])].cpu().numpy(), oo

        enqueue()
        return d_v, finish

    def run(self, units: Sequence, parts: List[List[int]], stage_mask: int, unit_stages=None, toon_flags: int = 0, mask_max_depth: int = 10):
        import torch
        import torch.distributed as dist

        mine = parts[self.rank]
        words = self.engine.VERDICT_DTYPE.itemsize // 8
        counts = [len(p) for p in parts]
        dev = torch.device("cuda", self.device) if self.backend == "nccl" else torch.device("cpu")
        us = None if unit_stages is None or not mine else np.asarray(unit_stages, dtype=np.uint8)[mine]
        # NCCL with the GPU chain: verdict records stay on the device, the all-gather runs on the chain's stream, the host copy comes
        # after the collective
        on_device = bool(mine) and self.backend == "nccl" and type(self)._local is ShardedChain._local
        finish = None
        if on_device:
            local, finish = self._enqueue_device([units[i] for i in mine], stage_mask, us, toon_flags, words, mask_max_depth)
        else:
            if mine:
                # the depth only when masking is asked for, so that an override of _local without masking keeps its signature
                depth = {"mask_max_depth": mask_max_depth} if stage_mask & CF_STAGE_MASK else {}
                v, out, oo = self._local([units[i] for i in mine], stage_mask, us, toon_flags, **depth)
            else:
                v, out, oo = np.zeros(0, dtype=self.engine.VERDICT_DTYPE), np.zeros(0, dtype=np.uint8), np.zeros(1, dtype=np.uint64)
            local = torch.from_numpy(np.ascontiguousarray(v).view(np.int64).copy()).to(dev)
        # one collective: verdict records as int64 triples, padded to the largest shard
        gathered = gather_verdicts(local, counts, words, self.group)
        if finish is not None:
            out, oo = finish()
        full = np.zeros(len(units), dtype=self.engine.VERDICT_DTYPE)
        for idxs, t in zip(parts, gathered):
            if idxs:
                full[np.asarray(idxs)] = t.cpu().numpy().view(self.engine.VERDICT_DTYPE)
        return full, mine, out, oo
