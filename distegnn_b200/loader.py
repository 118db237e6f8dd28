"""Loader around the shard format (SURVEY §8 f-4): PyG-`DataLoader` collation + pinned prefetch, CSR all the way.

The reference feeds its model through `torch_geometric.loader.DataLoader(dataset, batch_size, drop_last=True,
num_workers=4, sampler=RandomSampler(dataset, generator=Generator().manual_seed(seed)))` (main.py:178-190): every rank
draws the SAME permutation (same-seed sampler) and loads its own partition of those graphs; PyG's collation concatenates
the node tensors of the `batch_size` graphs, offsets `edge_index` by the running node count and emits the `batch` vector;
the model then sorts the int64 edges.  Here:

  * `collate(shards)`  — the same collation on pre-sorted CSR shards: node arrays concatenated, `rowptr` / `col` offset by
    the running edge / node counts (graphs are disjoint, so the concatenation of per-graph CSRs IS the batch's CSR: nothing
    is sorted), `edge_attr` concatenated in CSR order, `data_batch` = graph id per node, `loc_mean` / `target` stacked;
  * `ShardLoader`      — an iterator over a list of shard files with the reference's sampling (same-seed `RandomSampler`
    without replacement for training, file order otherwise, `drop_last`), a background thread that reads + collates the
    next batches into PINNED staging buffers and issues their H2D copies on a side stream, and per-batch CUDA events, so
    the copy of batch i+1 overlaps the step on batch i.  It yields `(forward_kwargs, extras)`: the keyword arguments of
    `FastEGNN.forward` (`edge_index` = a `CSRGraph` on the device) and `extras` = {target, ptr (host ints), n_graphs}.
"""
from __future__ import annotations

import queue
import threading
from typing import Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import torch

from .shards import CSRGraph, Shard, read_shard

Tensor = torch.Tensor
_NODE_KEYS = ("node_feat", "node_loc", "node_vel", "node_attr", "target")


def collate(shards: Sequence[Shard]) -> Dict[str, Tensor]:
    """PyG `Batch.from_data_list` semantics on CSR shards (host tensors in, host tensors out).  Every input shard holds one
    graph (`data_batch` all zero) or an already collated batch (graph ids are offset by the running graph count)."""
    out: Dict[str, List[Tensor]] = {}
    n_off, e_off, g_off = 0, 0, 0
    ptr = [0]
    rowptrs, cols, batches = [], [], []
    for sh in shards:
        t = sh.t
        n, e = int(t["node_loc"].shape[0]), int(t["col"].shape[0])
        for k in _NODE_KEYS:
            if k in t:
                out.setdefault(k, []).append(t[k])
        if "edge_attr" in t:
            out.setdefault("edge_attr", []).append(t["edge_attr"])
        out.setdefault("loc_mean", []).append(t["loc_mean"])
        rp = t["rowptr"].to(torch.int64)
        rowptrs.append((rp[:-1] if len(rowptrs) < len(shards) - 1 else rp) + e_off)
        cols.append(t["col"].to(torch.int64) + n_off)
        b = t["data_batch"].to(torch.int64)
        batches.append(b + g_off)
        ng = int(t["loc_mean"].shape[0])
        if ng == 1:
            ptr.append(n_off + n)
        else:                                                # an already collated shard: recover its graph boundaries
            cnt = torch.bincount(b, minlength=ng)
            for c in torch.cumsum(cnt, 0).tolist():
                ptr.append(n_off + int(c))
        n_off, e_off, g_off = n_off + n, e_off + e, g_off + ng
    if e_off >= 2 ** 31 or n_off >= 2 ** 31:
        raise ValueError("collated batch exceeds the int32 index range of the kernels")
    res = {k: torch.cat(v, 0) for k, v in out.items()}
    res["rowptr"] = torch.cat(rowptrs).to(torch.int32)
    res["col"] = torch.cat(cols).to(torch.int32)
    res["data_batch"] = torch.cat(batches).to(torch.int32)
    res["ptr"] = torch.tensor(ptr, dtype=torch.int64)
    return res


def batch_to_device(host: Dict[str, Tensor], device, non_blocking: bool = True) -> Tuple[Dict[str, object], Dict[str, object]]:
    """Collated host batch -> (FastEGNN.forward kwargs on `device`, extras)."""
    d = {k: v.to(device, non_blocking=non_blocking) for k, v in host.items() if k != "ptr"}
    graph = CSRGraph(d["rowptr"], d["col"])
    graph._checked = True                                    # produced by `collate` from CSR shards: valid by construction
    kwargs = dict(node_feat=d["node_feat"], node_loc=d["node_loc"], node_vel=d["node_vel"], loc_mean=d["loc_mean"],
                  edge_index=graph, data_batch=d["data_batch"].to(torch.int64),
                  edge_attr=d.get("edge_attr"), node_attr=d.get("node_attr"))
    ptr = host["ptr"].tolist()
    extras = dict(target=d.get("target"), ptr=ptr, n_graphs=len(ptr) - 1,
                  node_counts=[ptr[i + 1] - ptr[i] for i in range(len(ptr) - 1)])
    return kwargs, extras


class ShardLoader:
    """Iterate over shard files in batches, the reference's way (main.py:178-190), with pinned, overlapped H2D.

    paths       one shard file per graph (this rank's partition of it)
    batch_size  graphs per batch (`config.data.batch_size`)
    shuffle     True = `RandomSampler(replacement=False)` with a generator seeded by `seed` — every rank passes the same
                seed and therefore walks the graphs in the same order (the reference asserts exactly that, train.py:52-61)
    drop_last   as the reference (True)
    prefetch    batches staged ahead by the background thread (0 = synchronous, no thread)
    """

    def __init__(self, paths: Sequence[str], batch_size: int = 1, shuffle: bool = False, seed: int = 0,
                 drop_last: bool = True, device: Optional[torch.device] = None, prefetch: int = 2, pin_memory: bool = True):
        self.paths = list(paths)
        self.batch_size, self.shuffle, self.drop_last = int(batch_size), shuffle, drop_last
        self.device = torch.device(device) if device is not None else None
        self.prefetch, self.pin = int(prefetch), pin_memory and self.device is not None and self.device.type == "cuda"
        self.generator = torch.Generator()
        self.generator.manual_seed(seed)

    def __len__(self) -> int:
        return n_batches(len(self.paths), self.batch_size, self.drop_last)

    def _host_batch(self, idx: Sequence[int]) -> Dict[str, Tensor]:
        host = collate([read_shard(self.paths[i]) for i in idx])
        if self.pin:
            host = {k: (v if k == "ptr" else v.pin_memory()) for k, v in host.items()}
        return host

    def __iter__(self) -> Iterator[Tuple[Dict[str, object], Dict[str, object]]]:
        batches = sampler_batches(len(self.paths), self.batch_size, self.shuffle, self.generator, self.drop_last)
        if self.device is None or self.device.type != "cuda":
            for b in batches:
                yield batch_to_device(self._host_batch(b), self.device or "cpu", non_blocking=False)
            return
        yield from staged(batches, self._host_batch, lambda host: batch_to_device(host, self.device), self.device,
                          self.prefetch)


def n_batches(n: int, batch_size: int, drop_last: bool) -> int:
    return n // batch_size if drop_last else (n + batch_size - 1) // batch_size


def sampler_batches(n: int, batch_size: int, shuffle: bool, generator: torch.Generator,
                    drop_last: bool) -> List[List[int]]:
    """One epoch's batches of item indices: `RandomSampler(replacement=False)` order drawn from `generator` (every rank
    seeds it alike and walks the items in the same order) or index order, cut into `batch_size` batches, `drop_last`."""
    order = torch.randperm(n, generator=generator).tolist() if shuffle else list(range(n))
    batches = [order[i:i + batch_size] for i in range(0, len(order), batch_size)]
    if drop_last and batches and len(batches[-1]) < batch_size:
        batches.pop()
    return batches


def _record_on(v, stream) -> None:
    if isinstance(v, torch.Tensor):
        v.record_stream(stream)
    elif isinstance(v, CSRGraph):
        for t in (v.rowptr, v.col, v.row, v.info):
            if t is not None:
                t.record_stream(stream)


def staged(batches: Sequence, make_host: Callable, to_device: Callable, device: torch.device,
           prefetch: int) -> Iterator[Tuple[Dict[str, object], Dict[str, object]]]:
    """The loaders' staging pipeline on a CUDA device: a background thread builds each batch on the host
    (`make_host(batch)`, pinned buffers) and runs `to_device(host)` -> (kwargs, extras) on a side stream, so the H2D copy
    (and whatever device work `to_device` enqueues) of batch i+1 overlaps the step on batch i; one CUDA event per batch
    orders the consumer's stream after it.  prefetch = batches staged ahead (0 = synchronous, no thread)."""
    if prefetch <= 0:
        for b in batches:
            yield to_device(make_host(b))
        return
    copy_stream = torch.cuda.Stream(device=device)
    q: "queue.Queue" = queue.Queue(maxsize=prefetch)

    def worker():
        try:
            torch.cuda.set_device(device)
            for b in batches:
                host = make_host(b)
                with torch.cuda.stream(copy_stream):
                    item = to_device(host)
                    ev = torch.cuda.Event()
                    ev.record(copy_stream)
                q.put((item, ev, host))                      # `host` rides along: pinned memory must outlive the copy
            q.put(None)
        except BaseException as e:                           # noqa: BLE001 — surfaced on the consumer side
            q.put(e)

    th = threading.Thread(target=worker, daemon=True)
    th.start()
    while True:
        got = q.get()
        if got is None:
            break
        if isinstance(got, BaseException):
            raise got
        (kwargs, extras), ev, _host = got
        cur = torch.cuda.current_stream(device)
        cur.wait_event(ev)
        for v in list(kwargs.values()) + [extras.get("target")]:
            _record_on(v, cur)
        yield kwargs, extras
    th.join()
