"""Multi-GPU driver for the converter: replicas only (SURVEY.md section 8e).

Utterances are independent, so N GPUs = N replicas of the model, one process per GPU
(``torchrun``), no collective inside the hot path.  ``torch.distributed`` (NCCL over NVLink on
GPUs, gloo in the CPU tests) is used for exactly two things, as north_star prescribes:
broadcasting the checkpoint from rank 0 and gathering the output waveforms on rank 0.

Two gather paths: ``convert_sharded`` takes any ``convert_fn`` returning host arrays (host staging; what the CPU / gloo
tests drive), ``convert_sharded_async`` keeps the converted batch on the device, gathers it GPU-to-GPU (NCCL over
NVLink) on a side stream and copies it to pinned host memory on rank 0 only, so step i's gather and download overlap
step i+1's kernels.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist


def lpt_shard(costs: Sequence[float], world: int) -> List[List[int]]:
    """Longest-processing-time-first assignment of items (cost = samples) to ``world`` ranks.
    Deterministic; every rank computes the same table.  Returns per-rank index lists."""
    order = sorted(range(len(costs)), key=lambda i: (-costs[i], i))
    loads = [0.0] * world
    shards: List[List[int]] = [[] for _ in range(world)]
    for i in order:
        r = min(range(world), key=lambda q: (loads[q], q))
        shards[r].append(i)
        loads[r] += costs[i]
    return shards


def _world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def broadcast_state_dict(sd: Optional[Dict[str, torch.Tensor]], device: str = "cpu", src: int = 0) -> Dict[str, torch.Tensor]:
    """Rank ``src`` passes the checkpoint's state dict, the others pass None; everybody returns the
    same dict (CPU fp32 tensors).  One metadata broadcast + one flat tensor broadcast (~128 MB)."""
    rank, world = _world()
    if world == 1:
        assert sd is not None
        return sd
    meta = [None]
    if rank == src:
        names = sorted(sd)
        meta = [[(k, tuple(sd[k].shape)) for k in names]]
    dist.broadcast_object_list(meta, src=src)
    layout = meta[0]
    sizes = [int(np.prod(s)) if len(s) else 1 for _, s in layout]
    if rank == src:
        flat = torch.cat([sd[k].detach().float().reshape(-1) for k, _ in layout]).to(device)
    else:
        flat = torch.empty(sum(sizes), dtype=torch.float32, device=device)
    dist.broadcast(flat, src=src)
    flat = flat.cpu()
    out, o = {}, 0
    for (k, shape), n in zip(layout, sizes):
        out[k] = flat[o: o + n].reshape(shape).clone()
        o += n
    return out


def gather_waveforms(local: List[np.ndarray], local_idx: List[int], n_total: int, device: str = "cpu",
                     dst: int = 0) -> Optional[List[np.ndarray]]:
    """Gather variable-length float32 waveforms on rank ``dst`` in the original item order.
    Two fixed-shape collectives: lengths/indices table, then a padded [n_max, L_max] block."""
    rank, world = _world()
    if world == 1:
        out: List[Optional[np.ndarray]] = [None] * n_total
        for i, a in zip(local_idx, local):
            out[i] = a
        return out  # type: ignore[return-value]
    n_loc = len(local)
    stats = torch.tensor([n_loc, max([len(a) for a in local], default=0)], dtype=torch.int64, device=device)
    dist.all_reduce(stats, op=dist.ReduceOp.MAX)
    n_max, l_max = int(stats[0]), int(stats[1])
    table = torch.full((n_max, 2), -1, dtype=torch.int64, device=device)
    block = torch.zeros((n_max, max(l_max, 1)), dtype=torch.float32, device=device)
    for j, (i, a) in enumerate(zip(local_idx, local)):
        table[j, 0], table[j, 1] = i, len(a)
        block[j, : len(a)] = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)
    tables = [torch.empty_like(table) for _ in range(world)] if rank == dst else None
    blocks = [torch.empty_like(block) for _ in range(world)] if rank == dst else None
    dist.gather(table, tables, dst=dst)
    dist.gather(block, blocks, dst=dst)
    if rank != dst:
        return None
    out = [None] * n_total
    for t, b in zip(tables, blocks):
        t, b = t.cpu(), b.cpu()
        for j in range(n_max):
            i, n = int(t[j, 0]), int(t[j, 1])
            if i >= 0:
                out[i] = b[j, :n].numpy().copy()
    assert all(o is not None for o in out)
    return out  # type: ignore[return-value]


def _check_per_item_se(src_se, tgt_se) -> None:
    from .api import is_per_frame_se
    if is_per_frame_se(src_se) or is_per_frame_se(tgt_se):
        raise ValueError("sharded conversion takes one embedding per item, not a per-frame one or a ToneTrack")


def convert_sharded(convert_fn: Callable[..., List[np.ndarray]], audios: Sequence[np.ndarray], src_se, tgt_se,
                    device: str = "cpu", **kw) -> Optional[List[np.ndarray]]:
    """Every rank holds the same utterance list; each converts its LPT shard with ``convert_fn``
    (normally ``ToneColorConverter.convert_batch``) and rank 0 receives all results in order.
    ``src_se`` / ``tgt_se``: one embedding for all items, or a per-item sequence.  A per-item ``seeds`` or ``tau``
    keyword follows its utterance into the shard that converts it (``convert_fn`` receives the shard's values), so with
    ``seeds`` every result is independent of the world size.  Embeddings that vary over time are refused (ValueError)."""
    _check_per_item_se(src_se, tgt_se)
    rank, world = _world()
    shards = lpt_shard([len(a) for a in audios], world)
    mine = shards[rank]
    pick = (lambda se: [se[i] for i in mine]) if isinstance(src_se, (list, tuple)) else (lambda se: se)
    kw = _pick_per_item(kw, mine, len(audios))
    res = convert_fn([audios[i] for i in mine], pick(src_se),
                     [tgt_se[i] for i in mine] if isinstance(tgt_se, (list, tuple)) else tgt_se, **kw) if mine else []
    return gather_waveforms(res, mine, len(audios), device=device)


class ShardedJob:
    """Handle of one ``convert_sharded_async`` call.  ``result()`` blocks until rank ``dst`` holds every waveform in
    pinned host memory and returns them in the original order (views into a buffer that the second-next call on
    the same converter reuses; ``copy=True`` detaches them); the other ranks get ``None``."""

    def __init__(self, done, table, host, rank, dst, n_total, copy):
        self._done, self._table, self._host = done, table, host
        self._rank, self._dst, self._n, self._copy = rank, dst, n_total, copy

    def result(self) -> Optional[List[np.ndarray]]:
        if self._done is not None:
            self._done.synchronize()
        if self._rank != self._dst:
            return None
        out: List[Optional[np.ndarray]] = [None] * self._n
        for r, rows in enumerate(self._table):
            block = self._host[r]
            for j, (i, n) in enumerate(rows):
                a = block[j, :n]
                out[i] = a.copy() if self._copy else a
        assert all(o is not None for o in out)
        return out  # type: ignore[return-value]


def _pick_per_item(kw: dict, mine: List[int], n: int) -> dict:
    """``kw`` with its per-item ``seeds`` / ``tau`` sequences cut down to the items ``mine`` (checked against ``n``
    first, so every rank refuses the same malformed call)."""
    from .api import check_per_item, check_seeds
    kw = dict(kw)
    if kw.get("seeds") is not None:
        seeds = check_seeds(kw["seeds"], n)
        kw["seeds"] = [seeds[i] for i in mine]
    if "tau" in kw and np.ndim(kw["tau"]) != 0:
        taus = check_per_item(kw["tau"], n, "tau")[1]
        kw["tau"] = [taus[i] for i in mine]
    return kw


def convert_sharded_async(converter, audios: Sequence[np.ndarray], src_se, tgt_se, tau=0.3, dst: int = 0,
                          copy: bool = False, seeds: Optional[Sequence[int]] = None) -> ShardedJob:
    """Every rank holds the same utterance list; each enqueues its LPT shard with
    ``converter.convert_batch_device`` (no host sync), the padded result blocks are gathered on rank ``dst`` by
    ONE device-to-device collective on a side stream, and rank ``dst`` alone downloads them.  Shapes of every
    rank's block follow from the shared list, so no size exchange is needed.  Returns at once; call ``.result()``.
    ``src_se`` / ``tgt_se``: one embedding for all items, or a per-item sequence.  ``tau`` (scalar or per item) and
    ``seeds`` (one key per item) follow their utterance as in ``convert_sharded``.  Embeddings that vary over time are
    refused (ValueError)."""
    import torch
    _check_per_item_se(src_se, tgt_se)
    rank, world = _world()
    hop = converter.hps.data.hop_length
    samples = [len(a) // hop * hop for a in audios]
    shards = lpt_shard([len(a) for a in audios], world)
    n_max = max(len(sh) for sh in shards)
    # result blocks are as wide as the longest utterance's launch bucket (convert_batch_device pads to 16 hops), so a rank
    # whose shard holds it hands its result buffer to the gather without a copy
    l_max = -(-max(len(a) for a in audios) // (16 * hop)) * (16 * hop) if samples else 0
    mine = shards[rank]
    pick = (lambda se: [se[i] for i in mine]) if isinstance(src_se, (list, tuple)) else (lambda se: se)
    per = _pick_per_item({"tau": tau, "seeds": seeds}, mine, len(audios))
    state = converter.__dict__.setdefault("_shard_state", {"n": 0})
    k = state["n"] % 2
    state["n"] += 1
    # the converter's device-side result buffer of slot k is reused by this call: the gather / download of the job that
    # used it last (two calls ago) must have read it first
    last = state.get(f"done{k}")
    if last is not None and converter.device != "cpu" and torch.cuda.is_available():
        torch.cuda.current_stream(converter.device).wait_event(last)
    if mine:
        o, _ = converter.convert_batch_device([audios[i] for i in mine], pick(src_se),
                                              [tgt_se[i] for i in mine] if isinstance(tgt_se, (list, tuple)) else tgt_se,
                                              tau=per["tau"], slot=k,
                                              **({} if seeds is None else {"seeds": per["seeds"]}))
    else:
        o = torch.zeros(0, max(l_max, 1), dtype=torch.float32, device=converter.device)
    table = [[(i, samples[i]) for i in sh] for sh in shards]
    dev = o.device
    if world == 1:
        host = _pinned_block(state, f"h{k}", (1, max(n_max, 1), max(l_max, 1)), dev)
        done = None
        w = min(o.shape[1], host.shape[2])           # the device result is padded to the launch bucket (16 hops)
        if dev.type == "cuda":
            # download on a side stream: the next call's upload and kernels do not queue behind it
            side = state.get("side")
            if side is None:
                side = state["side"] = torch.cuda.Stream(dev)
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                side.wait_event(ready)
                if len(mine):
                    host[0, : o.shape[0], :w].copy_(o[:, :w], non_blocking=True)
                done = torch.cuda.Event()
                done.record(side)
            state[f"done{k}"] = done
        elif len(mine):
            host[0, : o.shape[0], :w].copy_(o[:, :w])
        return ShardedJob(done, table, host.numpy(), rank, dst, len(audios), copy)
    # fixed-shape block per rank (pad rows / columns), gathered on a side stream
    cuda = dev.type == "cuda"
    if cuda:
        side = state.get("side")
        if side is None:
            side = state["side"] = torch.cuda.Stream(dev)
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(dev))
    block = o
    if o.shape[0] != n_max or o.shape[1] != l_max:
        block = torch.zeros(n_max, max(l_max, 1), dtype=torch.float32, device=dev)
        w = min(o.shape[1], l_max)                   # the device result is padded to the launch bucket (16 hops)
        block[: o.shape[0], :w] = o[:, :w]
        if cuda:
            ready.record(torch.cuda.current_stream(dev))
    host = None
    done = None
    ctx = torch.cuda.stream(side) if cuda else _nullcontext()
    with ctx:
        if cuda:
            side.wait_event(ready)
            block.record_stream(side)
        blocks = [torch.empty_like(block) for _ in range(world)] if rank == dst else None
        dist.gather(block, blocks, dst=dst)
        if rank == dst:
            host = _pinned_block(state, f"h{k}", (world, n_max, max(l_max, 1)), dev)
            for r in range(world):
                host[r].copy_(blocks[r], non_blocking=True)
                if cuda:
                    blocks[r].record_stream(side)
        if cuda:
            done = torch.cuda.Event()
            done.record(side)
            state[f"done{k}"] = done
    return ShardedJob(done, table, host.numpy() if host is not None else None, rank, dst, len(audios), copy)


class _nullcontext:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


def _pinned_block(state, name, shape, dev):
    """Grow-only host buffers (pinned when the data comes from a GPU), two generations alternate."""
    import torch
    numel = int(np.prod(shape))
    buf = state.get(name)
    if buf is None or buf.numel() < numel:
        buf = torch.empty(int(numel * 1.1) + 1024, dtype=torch.float32)
        if dev.type == "cuda":
            buf = buf.pin_memory()
        state[name] = buf
    return buf[:numel].view(shape)
