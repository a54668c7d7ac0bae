"""Multi-GPU plumbing (torch.distributed; NCCL on GPUs, gloo in the CPU tests).

Both hot paths shard without any reduction:
  * sketching: units (files / records) are independent -> contiguous blocks of units per rank, no collective;
    sketches stay on the rank that made them (the host gathers them in input order to write a .msh).
  * dist all-vs-all: the REFERENCE axis is sharded per rank and stays resident; every rank owns the query tile made of
    its own sketches and broadcasts it to the others (the one exchange step).  Rank r then computes the
    [all queries] x [its references] block; the full query-major grid is the concatenation of the blocks along the
    reference axis (reference order of `mash dist`: CommandDistance.cpp:213-232).
Only tensor movement happens here; all arithmetic is in libmashgpu.so.
"""
import torch
import torch.distributed as td


def shard_bounds(n, world):
    """Contiguous block partition of n items over `world` ranks: [(begin, end)] per rank."""
    per = (n + world - 1) // world if world > 0 else n
    return [(min(n, r * per), min(n, (r + 1) * per)) for r in range(world)]


def exchange_query_tiles(hashes, n_hashes, lengths, counts=None, group=None):
    """Every rank broadcasts its tile of sketches (rows of `hashes`, with n_hashes / lengths); returns the
    concatenation over ranks in rank order, i.e. the global sketch order of `shard_bounds`.

    hashes: (m_r, s) int64/uint64 bit patterns, n_hashes: (m_r,) int32, lengths: (m_r,) int64. Tiles may have different
    row counts per rank (`counts` = list of row counts; gathered when None)."""
    world = td.get_world_size(group)
    rank = td.get_rank(group)
    dev = hashes.device
    if counts is None:
        c = torch.tensor([hashes.shape[0]], dtype=torch.int64, device=dev)
        allc = [torch.zeros_like(c) for _ in range(world)]
        td.all_gather(allc, c, group=group)
        counts = [int(x.item()) for x in allc]
    s = hashes.shape[1]
    out_h, out_n, out_l = [], [], []
    for r in range(world):
        if r == rank:
            bh, bn, bl = hashes.contiguous(), n_hashes.contiguous(), lengths.contiguous()
        else:
            bh = torch.empty((counts[r], s), dtype=hashes.dtype, device=dev)
            bn = torch.empty((counts[r],), dtype=n_hashes.dtype, device=dev)
            bl = torch.empty((counts[r],), dtype=lengths.dtype, device=dev)
        src = td.get_global_rank(group, r) if group is not None else r
        td.broadcast(bh, src=src, group=group)
        td.broadcast(bn, src=src, group=group)
        td.broadcast(bl, src=src, group=group)
        out_h.append(bh); out_n.append(bn); out_l.append(bl)
    return torch.cat(out_h), torch.cat(out_n), torch.cat(out_l), counts


BEST_INT_KEYS = ("n_hits", "n_total", "ref", "numer", "denom")
BEST_LIST_KEYS = ("ref", "numer", "denom", "distance", "pvalue")


def merge_best_lists(parts, n_best):
    """Best lists of several reference shards (dicts as DistJob.run_best returns them, as tensors, `ref` already global, the same Q
    and n_best in each) -> the best lists over all of them: hits ordered by (distance ascending, reference ascending), cut to
    n_best; entries past n_hits are zero.  n_total is the sum over the shards."""
    hits = torch.stack([p["n_hits"] for p in parts])                                    # (shards, Q)
    cols = {k: torch.cat([p[k] for p in parts], dim=1) for k in BEST_LIST_KEYS}         # (Q, shards * n_best)
    q, dev = hits.shape[1], hits.device
    rank = torch.arange(n_best, device=dev)
    valid = (rank.view(1, 1, -1) < hits.permute(1, 0).unsqueeze(2)).reshape(q, -1)
    # stable sort by reference, then by distance: ties in distance stay in reference order; invalid entries go last
    key_ref = torch.where(valid, cols["ref"], torch.full_like(cols["ref"], torch.iinfo(torch.int64).max))
    order = torch.sort(key_ref, dim=1, stable=True).indices
    key_d = torch.where(valid, cols["distance"], torch.full_like(cols["distance"], float("inf"))).gather(1, order)
    order = order.gather(1, torch.sort(key_d, dim=1, stable=True).indices)[:, :n_best]
    n_hits = torch.clamp(hits.sum(0), max=n_best)
    keep = rank.view(1, -1) < n_hits.view(-1, 1)
    out = {k: torch.where(keep, v.gather(1, order), torch.zeros_like(v[:, :n_best])) for k, v in cols.items()}
    out["n_hits"] = n_hits
    out["n_total"] = torch.stack([p["n_total"] for p in parts]).sum(0)
    return out


def merge_best(local, ref_begin, n_best, group=None):
    """Global best hits from per-shard ones.  With the reference axis sharded, DistJob.run_best on a rank yields each query's best
    list over that rank's references only; the union of the per-shard top n_best contains the global top n_best, so merging them
    under the same order rule (with GLOBAL reference indices) is exact.

    local: what run_best returned on this rank (numpy arrays or tensors; the same Q and n_best on every rank); ref_begin: global
    index of this rank's reference 0.  Returns the merged dict on every rank, as tensors on the device of the inputs (integers as
    int64)."""
    world = td.get_world_size(group)
    mine = {k: torch.as_tensor(v) for k, v in local.items()}
    mine = {k: v.to(torch.int64 if k in BEST_INT_KEYS else torch.float64).contiguous() for k, v in mine.items()}
    mine["ref"] = mine["ref"] + int(ref_begin)
    parts = [dict() for _ in range(world)]
    for k, v in mine.items():
        got = [torch.empty_like(v) for _ in range(world)]
        td.all_gather(got, v, group=group)
        for r in range(world):
            parts[r][k] = got[r]
    return merge_best_lists(parts, n_best)


def merge_component_labels(parts):
    """Component labels of a union of graphs on the same n vertices from the labels of each (tensors of n smallest-member labels,
    as DistJob.components returns them per reference shard) -> the labels of the union, label[i] = smallest vertex of i's component.

    Part r is a star forest i -> L_r[i], which has the components of graph r.  Min-label propagation with pointer jumping over the
    edges {i, L_r[i]} of all parts: every round hooks each root under the smallest root it is joined to, then flattens the forest
    until every vertex points at its root; at the fixed point no edge joins two labels.  Labels only ever move to a smaller vertex of
    the same component, so the fixed point is the smallest member of each.  Torch ops only: runs on the labels' device."""
    if not parts:
        raise ValueError("no label arrays to merge")
    parts = [torch.as_tensor(p).to(torch.int64) for p in parts]
    n, dev = parts[0].numel(), parts[0].device
    idx = torch.arange(n, dtype=torch.int64, device=dev)
    return _min_labels(n, torch.cat([idx] * len(parts)), torch.cat([p.to(dev).reshape(-1) for p in parts]), dev)


def _min_labels(n, src, dst, dev):
    """label[i] = smallest vertex of i's component in the graph on n vertices with the edges {src[e], dst[e]} (int64 tensors)"""
    lab = torch.arange(n, dtype=torch.int64, device=dev)
    while True:
        a, b = lab[src], lab[dst]
        m = torch.minimum(a, b)
        new = lab.clone()
        new.scatter_reduce_(0, a, m, "amin")
        new.scatter_reduce_(0, b, m, "amin")
        while True:
            jumped = new[new]
            if torch.equal(jumped, new):
                break
            new = jumped
        if torch.equal(new, lab):
            return lab
        lab = new


FOREST_KEYS = ("row", "col", "numer", "denom", "distance", "pvalue")


def merge_spanning_forests(parts, n):
    """Minimum spanning forest of the union of several edge sets on the same n vertices, from the minimum spanning forest of each
    (dicts as DistJob.spanning_forest returns them, `col` global, e.g. one per reference shard).  Exact: by the cycle property an edge
    that is not in its own part's forest is the largest of a cycle in the union, so the union of the parts' forests contains the
    forest of the union.  Edges are ranked once by (distance, col, row), the forest's strict order; Boruvka rounds on the rank then
    pick every component's cheapest edge with scatter_reduce and join the components with the min-label propagation of
    merge_component_labels.  Torch ops only: runs on the device of the parts, with no communication.  Returns the forest's edges in
    forest order as a dict of tensors (integers as int64)."""
    if not parts:
        raise ValueError("no forests to merge")
    cols = {k: torch.cat([torch.as_tensor(p[k]).reshape(-1).to(torch.float64 if k in ("distance", "pvalue") else torch.int64) for p in parts])
            for k in FOREST_KEYS}
    dev = cols["row"].device
    cols = {k: v.to(dev) for k, v in cols.items()}
    # rank = position in (distance, col, row) order: stable sorts from the last key to the first
    order = torch.sort(cols["row"], stable=True).indices
    order = order[torch.sort(cols["col"][order], stable=True).indices]
    order = order[torch.sort(cols["distance"][order], stable=True).indices]
    u, v = cols["row"][order], cols["col"][order]
    m = u.numel()
    rank = torch.arange(m, dtype=torch.int64, device=dev)
    chosen = torch.zeros(m, dtype=torch.bool, device=dev)
    lab = torch.arange(n, dtype=torch.int64, device=dev)
    while True:
        a, b = lab[u], lab[v]
        live = a != b
        if not bool(live.any()):
            break
        best = torch.full((n,), m, dtype=torch.int64, device=dev)
        best.scatter_reduce_(0, a[live], rank[live], "amin")
        best.scatter_reduce_(0, b[live], rank[live], "amin")
        chosen[best[best < m]] = True           # a mutual pick is one edge
        lab = _min_labels(n, u[chosen], v[chosen], dev)
    keep = order[chosen]
    return {k: c[keep] for k, c in cols.items()}


def spanning_forest(local, group=None):
    """Global minimum spanning forest from per-shard ones.  With the reference axis sharded, DistJob.spanning_forest of an encoded job on
    a rank yields the forest of that rank's edges; all ranks gather the shards' forests (at most n - 1 edges each) and merge them
    (merge_spanning_forests).  local: this rank's forest (numpy arrays or tensors).  Returns the global forest on every rank, as tensors
    on the device of the inputs (integers as int64)."""
    world = td.get_world_size(group)
    mine = {k: torch.as_tensor(local[k]).reshape(-1) for k in FOREST_KEYS}
    mine = {k: v.to(torch.float64 if k in ("distance", "pvalue") else torch.int64).contiguous() for k, v in mine.items()}
    dev = mine["row"].device
    counts = _all_gather(torch.tensor([mine["row"].numel()], dtype=torch.int64, device=dev), world, group).view(-1).tolist()
    top = max(counts)
    parts = [dict() for _ in range(world)]
    for k, v in mine.items():
        padded = torch.zeros(top, dtype=v.dtype, device=dev)
        padded[:v.numel()] = v
        got = _all_gather(padded, world, group)
        for r in range(world):
            parts[r][k] = got[r, :counts[r]]
    n = max((int(p["row"].max()) + 1 for p in parts if p["row"].numel()), default=0)     # vertices without an edge play no part
    return merge_spanning_forests(parts, n)


def merge_components(labels, group=None):
    """Global components from per-shard ones.  With the reference axis sharded, DistJob.components of an encoded job on a rank
    yields the components of that rank's edges over all sketches; the component graph is the union of the ranks' edge sets, so
    merging the label arrays is exact.  labels: this rank's (n,) labels (numpy or tensor; the same n on every rank).  Returns the
    global labels (int64) on every rank, on the device of the input."""
    world = td.get_world_size(group)
    mine = torch.as_tensor(labels).to(torch.int64).contiguous()
    return merge_component_labels(list(_all_gather(mine, world, group)))


class DictOps:
    """The four device steps of the sharded dictionary build, on torch tensors (C ABI: mashgpu_dict_*).  The CPU tests pass
    a stand-in with the same methods to exercise the exchange protocol under gloo."""

    def __init__(self, eng, stream=None):
        self.eng, self.stream = eng, stream

    def local_sort(self, hashes, n_hashes, sketch_size):
        m, stride = hashes.shape
        cap = m * min(stride, sketch_size + 1)
        keys = torch.empty(max(1, cap), dtype=torch.int64, device=hashes.device)
        slots = torch.empty(max(1, cap), dtype=torch.int32, device=hashes.device)
        n = self.eng.dict_local_sort(hashes.data_ptr(), n_hashes.data_ptr(), m, stride, sketch_size, keys.data_ptr(), slots.data_ptr(), self.stream)
        return keys[:n], slots[:n]

    def split(self, keys, splitters):
        return self.eng.dict_split(keys.data_ptr(), keys.numel(), splitters, self.stream)

    def rank(self, keys):
        codes = torch.empty(max(1, keys.numel()), dtype=torch.int32, device=keys.device)
        nd = self.eng.dict_rank(keys.data_ptr(), keys.numel(), codes.data_ptr(), self.stream)
        return codes[:keys.numel()], nd

    def scatter(self, codes, slots, seg_counts, seg_base, hashes, n_hashes, sketch_size):
        m, stride = hashes.shape
        rows = torch.empty((m, sketch_size + 1), dtype=torch.int32, device=hashes.device)
        n_eff = torch.empty((m,), dtype=torch.int32, device=hashes.device)
        self.eng.dict_scatter(codes.data_ptr(), slots.data_ptr(), seg_counts, seg_base, n_hashes.data_ptr(), m, stride, sketch_size,
                              rows.data_ptr(), n_eff.data_ptr(), self.stream)
        return rows, n_eff


def _sync(t):
    if t.is_cuda:
        torch.cuda.current_stream(t.device).synchronize()


def _all_gather(x, world, group=None):
    """all_gather_into_tensor in the one form both NCCL and gloo take (flat concatenation); returns (world,) + x.shape."""
    out = torch.empty((world * x.numel(),), dtype=x.dtype, device=x.device)
    td.all_gather_into_tensor(out, x.contiguous().view(-1), group=group)
    return out.view((world,) + tuple(x.shape))


def sharded_dictionary(ops, hashes, n_hashes, lengths, sketch_size, group=None, n_samples=2048):
    """Dictionary-encodes a collection whose rows are sharded over the ranks (this rank holds `hashes` (m, stride) int64 bit
    patterns of uint64 hashes, `n_hashes` (m,) int32, `lengths` (m,) int64; shard sizes may differ) WITHOUT any rank sorting
    the whole collection: a sample sort by hash range.

      1. every rank sorts its own hashes (ops.local_sort) and contributes evenly spaced samples; all ranks pick the same G-1
         splitters from the gathered samples;
      2. the sorted keys are cut at the splitters and exchanged (all-to-all): rank d receives hash range d of every rank;
      3. rank d ranks the distinct values of its range (ops.rank); the distinct counts are all-gathered, their exclusive
         prefix sum is the code offset of each range;
      4. the codes travel back (all-to-all), the owners scatter them into rows of sketch_size+1 codes (ops.scatter);
      5. rows, per-row counts and lengths are all-gathered: every rank ends with the whole encoded collection in global order
         (rank 0's rows first), 4 bytes per hash.

    Returns (rows (N, sketch_size+1) int32, n_eff (N,) int32, lengths (N,) int64, counts per rank, stats dict)."""
    world = td.get_world_size(group)
    rank = td.get_rank(group)
    dev = hashes.device
    m = hashes.shape[0]
    # 1. local sort + samples
    keys, slots = ops.local_sort(hashes, n_hashes, sketch_size)
    n = keys.numel()
    step = max(1, n // n_samples)
    samp = torch.full((n_samples,), -1, dtype=torch.int64, device=dev)        # -1 = 2^64-1 as a bit pattern: sorts last, never a splitter
    take = keys[::step][:n_samples]
    samp[:take.numel()] = take
    meta = torch.tensor([m, n], dtype=torch.int64, device=dev)
    all_samp = _all_gather(samp, world, group)
    all_meta = _all_gather(meta, world, group)
    all_meta_h = all_meta.cpu().numpy()
    counts = [int(x) for x in all_meta_h[:, 0]]
    # splitters: quantiles of the weighted sample (every rank's samples stand for step_r keys each)
    import numpy as np
    sh = all_samp.cpu().numpy().view(np.uint64)
    w = np.concatenate([np.full(n_samples, max(1, int(all_meta_h[r, 1]) // n_samples), np.int64) for r in range(world)])
    flat = sh.reshape(-1)
    valid = flat != np.uint64(0xFFFFFFFFFFFFFFFF)
    flat, w = flat[valid], w[valid]
    order = np.argsort(flat, kind="stable")
    flat, w = flat[order], w[order]
    cum = np.cumsum(w)
    splitters = np.empty(world - 1, np.uint64)
    for d in range(1, world):
        if flat.size == 0:
            splitters[d - 1] = np.uint64(0xFFFFFFFFFFFFFFFF)
        else:
            i = int(np.searchsorted(cum, cum[-1] * d / world))
            splitters[d - 1] = flat[min(i, flat.size - 1)]
    # 2. cut + exchange
    send_counts = ops.split(keys, splitters) if world > 1 else [n]
    sc = torch.tensor(send_counts, dtype=torch.int64, device=dev)
    all_sc = _all_gather(sc, world, group)
    all_sc_h = all_sc.cpu().numpy()
    recv_counts = [int(all_sc_h[r, rank]) for r in range(world)]
    recv = torch.empty((sum(recv_counts),), dtype=torch.int64, device=dev)
    _sync(keys)
    td.all_to_all_single(recv, keys.contiguous(), recv_counts, [int(c) for c in send_counts], group=group)
    _sync(recv)          # the library works on its own stream: the collective must have landed
    # 3. rank the distinct values of my hash range
    codes_r, n_distinct = ops.rank(recv)
    nd = torch.tensor([n_distinct], dtype=torch.int64, device=dev)
    all_nd_h = [int(x) for x in _all_gather(nd, world, group).cpu().numpy().reshape(-1)]
    base = [sum(all_nd_h[:d]) for d in range(world)]
    # 4. codes back to the owners, scatter into rows
    codes = torch.empty((n,), dtype=torch.int32, device=dev)
    _sync(codes_r)
    td.all_to_all_single(codes, codes_r.contiguous(), [int(c) for c in send_counts], recv_counts, group=group)
    _sync(codes)
    rows, n_eff = ops.scatter(codes, slots, [int(c) for c in send_counts], base, hashes, n_hashes, sketch_size)
    # 5. all-gather the encoded rows (shards padded to the largest)
    per = max(counts) if counts else 0
    P = sketch_size + 1

    def gather_rows(x, width, dtype):
        buf = torch.zeros((per,) + ((width,) if width else ()), dtype=dtype, device=dev)
        buf[:m] = x
        _sync(buf)
        out = _all_gather(buf, world, group).view((world * per,) + ((width,) if width else ()))
        if all(c == per for c in counts):
            return out
        return torch.cat([out[r * per:r * per + counts[r]] for r in range(world)])

    all_rows = gather_rows(rows, P, torch.int32)
    all_neff = gather_rows(n_eff, 0, torch.int32)
    all_len = gather_rows(lengths, 0, torch.int64)
    _sync(all_len)
    stats = {"keys_sorted_locally": n, "keys_ranked": int(recv.numel()), "distinct_total": sum(all_nd_h),
             "bytes_sent_all_to_all": int(8 * (n - send_counts[rank]) + 4 * (recv.numel() - recv_counts[rank])),
             "bytes_all_gather_rows": int(4 * P * sum(counts))}
    return all_rows, all_neff, all_len, counts, stats


def screen_allreduce(job, group=None):
    """Multi-GPU screen: reads are sharded over ranks, every rank holds the same reference table.  Sums the hit counters
    over ranks in place (NCCL all-reduce on the job's device counter array) and folds every rank's mixture bottom-s list into
    this rank's job on the device (one all-gather of G x s hashes, one merge kernel, no host round trip per rank), after which
    job.finish() returns the global result on every rank."""
    ptr, n_slots = job.counters()
    dev = torch.device("cuda", job.eng.device)

    class _Cai:        # expose the library's device buffers to torch without a copy (CUDA array interface)
        def __init__(self, p, n, typestr):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (p, False), "version": 3}

    if n_slots:
        counters = torch.as_tensor(_Cai(ptr, n_slots, "<i4"), device=dev)
        td.all_reduce(counters, op=td.ReduceOp.SUM, group=group)
    s = job.p.sketch_size
    mix_ptr, mix_n_ptr = job.mixture_dev()
    mine = torch.as_tensor(_Cai(mix_ptr, s, "<i8"), device=dev)
    mine_n = torch.as_tensor(_Cai(mix_n_ptr, 1, "<i4"), device=dev)
    world = td.get_world_size(group)
    all_lists = _all_gather(mine.clone(), world, group)
    all_counts = _all_gather(mine_n.clone(), world, group)
    torch.cuda.current_stream(dev).synchronize()     # the engine merges on its own stream
    job.merge_mixtures_dev(all_lists.data_ptr(), all_counts.data_ptr(), world, s)


def bind_to_gpu_numa_node(device_index):
    """Restrict this thread -- and every thread it creates afterwards: the engine's packer pool, its upload helper -- to the CPUs of
    the NUMA node the GPU hangs off, so that page-locked host buffers are first touched on that node and the DMA reads and the
    packer's reads do not cross the socket interconnect.  With 8 ranks per node every rank otherwise competes for both sockets'
    memory controllers.  Returns (node, n_cpus) or None when the topology is
    not visible (single node, a VM without NUMA information) or the affinity cannot be changed."""
    try:
        import os
        pr = torch.cuda.get_device_properties(device_index)
        bdf = "%04x:%02x:%02x.0" % (getattr(pr, "pci_domain_id", 0), pr.pci_bus_id, pr.pci_device_id)
        node = int(open(f"/sys/bus/pci/devices/{bdf}/numa_node").read())
        if node < 0:
            return None
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        allowed = os.sched_getaffinity(0) & cpus
        if not allowed:
            return None
        os.sched_setaffinity(0, allowed)
        return node, len(allowed)
    except (OSError, ValueError, AttributeError, RuntimeError, AssertionError):
        return None


def warm_collectives(dev, group=None):
    """First use of a collective on a fresh NCCL communicator sets up its channels (hundreds of ms for all-reduce over 8 ranks);
    a process pays that once at start-up, so the benchmarks run one small instance of each collective they time before timing."""
    world = td.get_world_size(group)
    x = torch.ones((world * 4,), dtype=torch.int64, device=dev)
    y = torch.empty_like(x)
    td.all_reduce(x, group=group)
    td.all_to_all_single(y, x, group=group)
    _all_gather(x, world, group)
    td.broadcast(x, src=td.get_global_rank(group, 0) if group is not None else 0, group=group)
    big = torch.zeros((1 << 24,), dtype=torch.int32, device=dev)          # 64 MB: the large-message all-reduce path too
    td.all_reduce(big, group=group)
    if dev.type == "cuda":
        torch.cuda.synchronize(dev)


def assemble_grid(blocks):
    """blocks[r]: (n_qry, n_ref_r) block computed by rank r -> (n_qry, n_ref) in global reference order."""
    return torch.cat(list(blocks), dim=1)
