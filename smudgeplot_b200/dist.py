"""One-process-per-GPU sharding of the hetmers scan (torch.distributed = plumbing; NCCL over
NVLink/NVSwitch on GPUs, gloo in the CPU tests of the host logic).

Path partition (DESIGN.md §6; SURVEY.md §8e): the sorted table is cut into `world` contiguous
shards on prefix-bucket boundaries ("canonical-prefix buckets" of BASELINE.json's north_star).
Rank r loads / owns shard r, every rank ends with a full replica (shards broadcast over NVLink),
and rank r scans index range [lo_r, hi_r):

    pass 1 (own range, lower pair member does the book-keeping)  -> partial incidence array
    all-reduce(sum, uint8[n])                                    <- the one real exchange step
    pass 2 (own range)                                           -> partial plot
    all-reduce(sum, int64[1001*501])                             <- the reference's serial
                                                                    plot reduction, :1569-1575
The reference has no multi-process code at all; its only "collective" is that final sum.
"""
from __future__ import annotations

import os
import time

import torch
import torch.distributed as dist


def prefix_partition(world: int, bits: int = 24):
    """equal split of the `bits`-bit prefix space: [(lo_r, hi_r)] for r in range(world)"""
    top = 1 << bits
    return [((top * r) // world, (top * (r + 1)) // world) for r in range(world)]


def shard_offsets(local_n: int, group=None, device=None):
    """all ranks' shard sizes -> (sizes list, offsets list, total)"""
    world = dist.get_world_size(group)
    t = torch.zeros(world, dtype=torch.int64, device=device)
    t[dist.get_rank(group)] = local_n
    dist.all_reduce(t, group=group)
    sizes = [int(x) for x in t.tolist()]
    offs = [0]
    for s in sizes:
        offs.append(offs[-1] + s)
    return sizes, offs[:-1], offs[-1]


def _exchange_to_even_chunks(buf: torch.Tensor, sizes, offs, chunk: int, total: int, group=None):
    """buf (padded to world*chunk elements) holds this rank's shard [offs[r], offs[r]+sizes[r]) in place; afterwards
    it also holds everything of the even chunk [r*chunk, (r+1)*chunk): the slivers that belong to that chunk but
    were loaded by other ranks arrive by point-to-point copies (shards of a prefix partition are nearly even, so
    the slivers are small)"""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    ops, keep = [], []
    for q in range(world):
        oq0, oq1 = offs[q], offs[q] + sizes[q]
        for r in range(world):
            if q == r:
                continue
            a, b = max(oq0, r * chunk), min(oq1, min((r + 1) * chunk, total))
            if a >= b or rank not in (q, r):
                continue
            peer = r if rank == q else q
            peer = dist.get_global_rank(group, peer) if group is not None else peer
            t = buf[a:b]
            keep.append(t)
            ops.append(dist.P2POp(dist.isend if rank == q else dist.irecv, t, peer, group))
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()


def gather_table(local_keys: torch.Tensor, local_cnt: torch.Tensor, group=None, out=None,
                 local_lo: torch.Tensor | None = None, out_lo: torch.Tensor | None = None):
    """Assemble the full sorted table on every rank from per-rank shards (shard r = rank r's
    slice of the key space, so concatenation in rank order is the sorted table): the shards are evened
    out by small point-to-point copies and then ONE all-gather per array moves everything (instead of
    3 x world sequential broadcasts).
    -> (keys_full, cnt_full, lo, hi) with [lo,hi) this rank's index range; with `local_lo` (second
    key word, k > 32) -> (keys_full, cnt_full, lo, hi, keys_lo_full).
    `out` buffers are used in place when they have room for world*ceil(total/world) elements."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    sizes, offs, total = shard_offsets(local_keys.numel(), group, local_keys.device)
    chunk = (total + world - 1) // world if world > 0 else total
    padded = max(chunk * world, total)

    def room(t, dtype, device):
        if t is not None and t.numel() >= padded:
            return t
        return torch.empty(padded, dtype=dtype, device=device)

    kbuf = room(out[0] if out is not None else None, local_keys.dtype, local_keys.device)
    cbuf = room(out[1] if out is not None else None, local_cnt.dtype, local_cnt.device)
    lbuf = room(out_lo, local_lo.dtype, local_lo.device) if local_lo is not None else None
    lo, hi = offs[rank], offs[rank] + sizes[rank]
    pairs = [(kbuf, local_keys), (cbuf, local_cnt)] + ([(lbuf, local_lo)] if lbuf is not None else [])
    for buf, loc in pairs:
        if loc.numel() and loc.data_ptr() != buf[lo:hi].data_ptr():
            buf[lo:hi].copy_(loc)
    if world > 1 and total > 0:
        for buf, _ in pairs:
            raw = buf.view(torch.uint8)                     # counts travel as raw bytes (gloo has no int16 collectives)
            w = buf.element_size()
            _exchange_to_even_chunks(raw, [s_ * w for s_ in sizes], [o * w for o in offs], chunk * w, total * w, group)
            own = raw[rank * chunk * w:(rank + 1) * chunk * w].clone()
            try:
                dist.all_gather_into_tensor(raw[:world * chunk * w], own, group=group)
            except (RuntimeError, NotImplementedError):
                parts = [torch.empty_like(own) for _ in range(world)]
                dist.all_gather(parts, own, group=group)
                for r, pt in enumerate(parts):
                    raw[r * chunk * w:(r + 1) * chunk * w].copy_(pt)
    keys, cnt = kbuf[:total], cbuf[:total]
    if out is not None:                                      # caller's buffers too small for the padding: copy back
        if out[0].data_ptr() != kbuf.data_ptr():
            out[0][:total].copy_(keys)
            keys = out[0][:total]
        if out[1].data_ptr() != cbuf.data_ptr():
            out[1][:total].copy_(cnt)
            cnt = out[1][:total]
    if lbuf is not None:
        klo = lbuf[:total]
        if out_lo is not None and out_lo.data_ptr() != lbuf.data_ptr():
            out_lo[:total].copy_(klo)
            klo = out_lo[:total]
        return keys, cnt, lo, hi, klo
    return keys, cnt, lo, hi


def _cuda_view(ptr: int, nbytes: int, device) -> torch.Tensor:
    """uint8 tensor over a raw device allocation (no ownership) via __cuda_array_interface__"""
    class _Raw:
        pass
    r = _Raw()
    r.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}
    return torch.as_tensor(r, device=device)


def allreduce_deg(deg: torch.Tensor, group=None):
    """sum of the partial incidence arrays (uint8; no wrap: <= 3k <= 192 neighbours for k <= 64)"""
    dist.all_reduce(deg, op=dist.ReduceOp.SUM, group=group)
    return deg


def allreduce_plot(plot: torch.Tensor, group=None):
    dist.all_reduce(plot, op=dist.ReduceOp.SUM, group=group)
    return plot


def balanced_offsets(keys_full: torch.Tensor, world: int, depth: int = 3, per_candidate: float = 0.03):
    """Work ranges [off[r], off[r+1]) with equal pass-1 WORK rather than equal entry counts.
    Only neighbours y > x are probed, so an entry with base b at position p has 3-b candidates
    there ('a' three, 't' none) -- each ~3 % of an entry's cost.  For the first `depth` bases that
    number is the same for whole stretches of the sorted table, so shards cut by count are
    systematically uneven.  The table is split into the 4^depth prefix classes, each
    weighted by its candidate count, and the cuts are placed on the cumulative weight."""
    n = keys_full.numel()
    if world <= 1:
        return [0, n]
    sign = -(1 << 63)
    ncls = 4 ** depth
    flipped = keys_full ^ sign                                   # unsigned order as signed
    marks = []
    for c in range(1, ncls):
        v = c << (64 - 2 * depth)                                # first key of prefix class c (unsigned)
        v = v - (1 << 64) if v >= (1 << 63) else v               # as the int64 bit pattern
        marks.append(v ^ sign)
    pos = torch.searchsorted(flipped, torch.tensor(marks, dtype=torch.int64, device=keys_full.device))
    bnd = [0] + [int(v) for v in pos.tolist()] + [n]
    w = []
    for c in range(ncls):
        cand = sum(3 - ((c >> (2 * (depth - 1 - p))) & 3) for p in range(depth))
        w.append(1.0 + per_candidate * cand)
    total = sum(w[c] * (bnd[c + 1] - bnd[c]) for c in range(ncls))
    offs, acc, c, at = [0], 0.0, 0, 0
    for r in range(1, world):
        target = total * r / world
        while c < ncls and acc + w[c] * (bnd[c + 1] - at) < target:
            acc += w[c] * (bnd[c + 1] - at)
            c += 1
            at = bnd[c] if c < ncls else n
        if c >= ncls:
            offs.append(n)
            continue
        step = int((target - acc) / w[c])
        acc += w[c] * step
        at += step
        offs.append(min(max(at, offs[-1]), n))
    return offs + [n]


def run_aligned_cuts(keys_full: torch.Tensor, kmer: int, world: int):
    """Shard cuts of the strand-symmetric scan: equal entry counts, each cut moved to the next RUN
    boundary (a run = entries sharing their first k/2 bases; all partners the run scan looks for lie in
    one run, so no pair straddles two shards).  Pure torch: every rank computes the same cuts from its
    replica.  -> [0, c1, ..., n]"""
    n = keys_full.numel()
    sh = 64 - 2 * (kmer >> 1)

    def pre(t):                                   # first k/2 bases as a non-negative number
        return (t >> sh) & ((1 << (64 - sh)) - 1) if sh > 0 else t

    cuts = [0]
    for r in range(1, world):
        c = max((n * r) // world, cuts[-1])
        if 0 < c < n:
            p0 = pre(keys_full[c - 1:c])
            while c < n:
                w = keys_full[c:c + 65536]
                d = torch.nonzero(pre(w) != p0)
                if d.numel():
                    c += int(d[0])
                    break
                c += w.numel()
        cuts.append(min(c, n))
    return cuts + [n]


def fingerprint_verdict(acc: torch.Tensor, group=None) -> bool:
    """acc = this rank's int64[4] fingerprint sums (device.DeviceTable.fingerprint over the entries it
    loaded, same seeds on every rank): symmetric iff the job-wide sums (mod 2^64) of {(x,cnt)} and
    {(rc x,cnt)} agree"""
    world = dist.get_world_size(group)
    parts = [torch.zeros_like(acc) for _ in range(world)]
    dist.all_gather(parts, acc, group=group)
    tot = [0, 0, 0, 0]
    for p in parts:
        for i, v in enumerate(p.tolist()):
            tot[i] = (tot[i] + v) & 0xFFFFFFFFFFFFFFFF
    return tot[0] == tot[2] and tot[1] == tot[3]


def common_seeds(device, group=None):
    """rank 0's fingerprint seeds for everybody"""
    import ctypes as C
    from . import _lib
    sd = (C.c_uint64 * 2)()
    _lib.lib().hm_symm_seeds(sd)
    t = torch.tensor([sd[0] - (1 << 64) if sd[0] >= (1 << 63) else sd[0],
                      sd[1] - (1 << 64) if sd[1] >= (1 << 63) else sd[1]], dtype=torch.int64, device=device)
    src = dist.get_global_rank(group, 0) if group is not None else 0
    dist.broadcast(t, src=src, group=group)
    return [int(v) & 0xFFFFFFFFFFFFFFFF for v in t.tolist()]


def exchange_segments(seg: torch.Tensor, rank: int, group=None):
    """seg[world, m]: row `rank` is this rank's Bloom segment; fill in everybody else's (all-gather)"""
    own = seg[rank].clone()
    try:
        dist.all_gather_into_tensor(seg.view(-1), own, group=group)
    except (RuntimeError, NotImplementedError):
        parts = [torch.empty_like(own) for _ in range(seg.shape[0])]
        dist.all_gather(parts, own, group=group)
        for r, p in enumerate(parts):
            seg[r].copy_(p)
    return seg


class PeerDeg:
    """The sharded incidence array of DESIGN.md §6 for a one-process-per-GPU job: every rank
    cudaMallocs its own full-length array through the C ABI (hm_dev_alloc), exports a CUDA IPC
    handle, and maps everybody else's (hm_ipc_open).  With it the exchange between the passes is
    fused into the kernels (remote atomics / remote loads over NVLink) and no collective moves the
    array.  `PeerDeg.create` returns None when IPC or native NVLink atomics are unavailable, and
    the caller falls back to the dense all-reduce."""

    def __init__(self, own, peers, nbytes, rank):
        self.own, self.peers, self.nbytes, self.rank = own, peers, nbytes, rank

    @classmethod
    def create(cls, n, device, group=None):
        import ctypes as C
        import os
        from . import _lib
        if os.environ.get("HETMERS_DENSE_EXCHANGE"):
            return None
        L = _lib.lib()
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        nbytes = (n + 256) & ~255               # one buffer; the allocation holds TWO (see scan_on)
        ok = 1
        own = C.c_void_p()
        handle = C.create_string_buffer(64)
        with torch.cuda.device(device):
            if L.hm_dev_alloc(2 * nbytes, C.byref(own)) != 0 or L.hm_ipc_export(own, handle) != 0:
                ok = 0
        info = [None] * world
        dist.all_gather_object(info, (ok, handle.raw, torch.cuda.current_device() if device.index is None else device.index),
                               group=group)
        peers = [None] * world
        if all(i[0] for i in info):
            for r, (_, h, dev_r) in enumerate(info):
                if r == rank:
                    peers[r] = own.value
                    continue
                if not L.hm_p2p_native_atomics(device.index or 0, dev_r):
                    ok = 0
                    break
                ptr = C.c_void_p()
                with torch.cuda.device(device):
                    if L.hm_ipc_open(h, C.byref(ptr)) != 0:
                        ok = 0
                        break
                peers[r] = ptr.value
        else:
            ok = 0
        flag = torch.tensor([ok], dtype=torch.int32, device=device)
        _in_place(lambda x: dist.all_reduce(x, op=dist.ReduceOp.MIN, group=group), flag, group)
        if int(flag.item()) == 0:
            with torch.cuda.device(device):
                for r, pp in enumerate(peers):
                    if pp is not None and r != rank:
                        L.hm_ipc_close(C.c_void_p(pp))
                if own.value:
                    L.hm_dev_free(own)
            return None
        return cls(own.value, peers, nbytes, rank)

    def close(self, device):
        """unmap the peers' arrays and free the own one (call on every rank, after a barrier)"""
        import ctypes as C
        from . import _lib
        L = _lib.lib()
        with torch.cuda.device(device):
            for r, pp in enumerate(self.peers):
                if pp is not None and r != self.rank:
                    L.hm_ipc_close(C.c_void_p(pp))
            if self.own:
                L.hm_dev_free(C.c_void_p(self.own))
        self.peers, self.own = [], None

    def shards(self, offsets, parity):
        """hm_shards over buffer `parity` (0/1) of every rank's allocation"""
        from . import _lib
        sh = _lib.Shards()
        sh.n_shards, sh.self_ = len(self.peers), self.rank
        for r, o in enumerate(offsets):
            sh.off[r] = o
        for r, pp in enumerate(self.peers):
            sh.deg[r] = pp + parity * self.nbytes
        return sh


class ShardedScan:
    """device-resident replica + this rank's work range; `scan()` = T_scan of SURVEY.md §8d, `extract()` =
    extract_kmer_pairs' list of the same job.  The collectives run on NCCL with a GPU per rank, or on gloo
    through host copies (several ranks may then share one GPU)."""

    def __init__(self, kmer, keys_full, cnt_full, lo, hi, group=None, keys_lo_full=None, path="auto"):
        import os
        from .device import DeviceTable
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self._coll_dev = keys_full.device if _nccl(group) else torch.device("cpu")
        self._backend = "NCCL" if _nccl(group) else "gloo, through host memory"
        self.table = DeviceTable(kmer, keys_full, cnt_full, keys_lo=keys_lo_full).build_index(direct=False)
        self.load_lo, self.load_hi = lo, hi       # the shard this rank LOADED (equal prefix ranges)
        self.kmer = kmer
        self.n_total = keys_full.numel()
        self.bits = self.table.bits
        self.peer = None
        self.stats = {}
        self._scanned = False                     # the last scan_on() was a scan() of self.table
        # is the whole table strand-symmetric?  every rank fingerprints the shard it loaded
        path = os.environ.get("HETMERS_PATH", path)
        self.seeds = common_seeds(self._coll_dev, group)
        self.symmetric = kmer >= 2 and fingerprint_verdict(
            self.table.fingerprint(lo, hi, self.seeds).to(self._coll_dev), group)
        self.table.symmetric = self.symmetric
        self.path = "symm" if (self.symmetric and path != "direct") else "direct"
        if self.path == "symm":
            # strand-symmetric scan: run-aligned shards of equal size, Bloom segments all-gathered
            self.offsets = run_aligned_cuts(keys_full, kmer, self.world)
            lo, hi = self.offsets[self.rank], self.offsets[self.rank + 1]
            self.table.alloc_symm(lo, hi, self.table.make_symm_shards(self.offsets, self.rank) if self.world > 1 else None)
            self.lo, self.hi = lo, hi
            self.exchange = f"all-gather of Bloom segments ({self._backend}) between run scan and resolve" \
                if self.world > 1 else "none"
        else:
            self._init_direct(keys_full)
        self._barrier_t = torch.zeros(1, dtype=torch.int32, device=keys_full.device)
        self._step = 0
        if keys_full.is_cuda:
            self._side = torch.cuda.Stream(device=keys_full.device)
        if self.peer is not None:       # tensors over the two halves of the IPC allocation (no ownership)
            self._peer_views = [_cuda_view(self.peer.own + h * self.peer.nbytes, self.peer.nbytes, keys_full.device)
                                for h in (0, 1)]

    def _init_direct(self, keys_full):
        """direct passes (any table): work-balanced shards, incidence array sharded by owner"""
        self.table.build_filter()
        # the shard this rank SCANS and owns the incidence bytes of: equal work, not equal counts
        self.offsets = balanced_offsets(keys_full, self.world)
        lo, hi = self.offsets[self.rank], self.offsets[self.rank + 1]
        self.table.alloc_work(lo, hi)
        self.lo, self.hi = lo, hi
        self.peer = PeerDeg.create(self.n_total, keys_full.device, self.group) if self.world > 1 else None
        self.exchange = "peer-memory (remote atomics/loads over NVLink, CUDA IPC)" if self.peer else \
                        (f"all-reduce(uint8[n]) via {self._backend}" if self.world > 1 else "none")

    @classmethod
    def from_synthetic(cls, k, G, ploidy, het, cov, L, seed, device, group=None):
        """every rank generates only its prefix-range shard of the seeded table, then the shards
        are exchanged (same flow as loading 1/world of the part files per rank)."""
        from tools import synth
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        rng = prefix_partition(world)[rank]
        keys, cnt = synth.synth_table(k, G, ploidy, het, cov, L, seed, device=device, key_range=rng)
        cnt16 = cnt.to(torch.int16)
        del cnt
        if k > 32:                               # two key words per k-mer
            khi, klo = keys[:, 0].contiguous(), keys[:, 1].contiguous()
            kf, cf, lo, hi, lf = gather_table(khi, cnt16, group, local_lo=klo)
            return cls(k, kf, cf, lo, hi, group, keys_lo_full=lf)
        kf, cf, lo, hi = gather_table(keys, cnt16, group)
        del keys, cnt16
        return cls(k, kf, cf, lo, hi, group)

    @classmethod
    def from_ktab(cls, name, group=None, device=None, path="auto", L=None, budget=None):
        """the FastK table `name` (stub + part files): rank r reads the records of ordinals [n*r/W, n*(r+1)/W)
        (a range may span part files), unpacks them on its GPU with the table's own ibyte, and the shares are
        all-gathered into the replica every rank holds (gather_table; on gloo the shares meet in host memory).
        With L (hetmers' -e) the table is first trimmed and / or symmetrised as hm_scan_examine(L) decides on the
        whole table, across the ranks (_from_ktab_conditioned, DESIGN.md §4e): the replica is what
        hetmers.Scan(kt).condition(L, not trimmed, not symmetric) + download() give in one process.  budget: device
        bytes per rank for that conditioning (default: free memory minus _lib.BUDGET_RESERVE)."""
        import numpy as np
        from . import fastk
        from .device import DeviceTable
        if L is not None:
            return cls._from_ktab_conditioned(name, group, device, path, int(L), budget)
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        dev = torch.device(device if device is not None else "cuda")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        kt = fastk.read_ktab(str(name), mmap=True)
        k, n = kt.kmer, kt.nels
        lo, hi = (n * rank) // world, (n * (rank + 1)) // world
        rec = _share_records(kt, lo, hi)
        with torch.cuda.device(dev):
            room = n + world                                   # room for gather_table's even chunks
            kb = torch.empty(room, dtype=torch.int64, device=dev)
            cb = torch.empty(room, dtype=torch.int16, device=dev)
            lb = torch.empty(room, dtype=torch.int64, device=dev) if k > 32 else None
            if hi > lo:
                d_rec = torch.from_numpy(rec).to(dev)
                d_idx = torch.from_numpy(np.ascontiguousarray(kt.index, dtype=np.int64)).to(dev)
                DeviceTable.from_records(k, kt.ibyte, d_rec, d_idx, first=lo, out=(kb, cb), out_lo=lb)
                del d_rec, d_idx
            del rec, kt
            share = (kb[lo:hi], cb[lo:hi], lb[lo:hi] if lb is not None else None)
            if _nccl(group):
                got = gather_table(share[0], share[1], group, out=(kb, cb), local_lo=share[2], out_lo=lb)
            else:
                got = gather_table(share[0].cpu(), share[1].cpu(), group,
                                   local_lo=share[2].cpu() if lb is not None else None)
                kb[:n].copy_(got[0])
                cb[:n].copy_(got[1])
                if lb is not None:
                    lb[:n].copy_(got[4])
            assert (got[2], got[3]) == (lo, hi)
            return cls(k, kb[:n], cb[:n], lo, hi, group, keys_lo_full=lb[:n] if lb is not None else None, path=path)

    @classmethod
    def _from_ktab_conditioned(cls, name, group, device, path, ethresh, budget):
        """from_ktab(L=ethresh): rank r loads its share of the source, the ranks decide "trimmed?" / "symmetric?"
        together (job_examine), and unless the table needs neither step every rank routes its kept entries (and
        their reverse complements) to the rank that owns their key prefix, which settles what it receives into its
        conditioned share (hm_k_shard_*); the shares are all-gathered into the replica.  The working set of every
        rank is checked against its budget once the summed histogram gives the counts, before any entry moves:
        HM_ENOMEM (or HM_EUNSUPPORTED, k > 32 and 2^32 - 16 reverse complements or more on one rank) on every
        rank, with the sizes.  stats["condition"]: verdicts, steps, entries in / out, entries sent to / received
        from each rank, peak device bytes of the call (torch's allocator; its peak statistics are reset), the
        working set and budget, and ms per phase on this rank."""
        from . import _lib, fastk
        from .device import _ptr, _stream
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        dev = torch.device(device if device is not None else "cuda")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        coll = dev if _nccl(group) else torch.device("cpu")
        Lb = _lib.lib()
        ms = {}
        lap = _lapper(ms)

        def done(phase, t):                                    # the phase's kernels have finished
            torch.cuda.synchronize(dev)
            return lap(phase, t)

        with torch.cuda.device(dev):
            if budget is None:
                budget = torch.cuda.mem_get_info(dev)[0] - _lib.BUDGET_RESERVE
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            t = time.perf_counter()
            kt = fastk.read_ktab(str(name), mmap=True)
            k, n, ibyte = kt.kmer, kt.nels, kt.ibyte
            two = k > 32
            lo, hi = share_range(n, world, rank)
            m = hi - lo
            sk, sc, sl = _load_share(kt, lo, hi, dev)
            del kt
            t = done("load", t)

            def share_min(a, b):
                out = torch.full((1,), 0x8000, dtype=torch.int32, device=dev)
                _lib.check(Lb.hm_k_min_count(_ptr(sc), a, b, _ptr(out), _stream()))
                return int(out.item())

            trimmed, symmetric = job_examine(ethresh, k, n, sk, sl, share_min, group, coll)
            do_trim, do_symm = not trimmed, not symmetric
            t = lap("examine", t)
            st = {"trimmed": trimmed, "symmetric": symmetric,
                  "steps": (["trim"] if do_trim else []) + (["symmetrise"] if do_symm else []),
                  "entries_in": n, "sent": [0] * world, "received": [0] * world, "budget": budget,
                  "working_set_bytes": 0}
            if do_trim or do_symm:
                share = [sk, sc, sl]                           # handed over: a refusal frees it before it raises
                del sk, sc, sl
                sk, sc, sl = _condition_share(k, ibyte, m, share, ethresh if do_trim else 0, do_symm, budget, group,
                                              coll, st, done, t)
                t = time.perf_counter()
            if _nccl(group):
                got = gather_table(sk, sc, group, local_lo=sl)
            else:
                got = gather_table(sk.cpu(), sc.cpu(), group, local_lo=sl.cpu() if two else None)
                got = [g.to(dev) if isinstance(g, torch.Tensor) else g for g in got]
            del sk, sc, sl
            done("gather", t)
            st["peak_bytes"] = torch.cuda.max_memory_allocated(dev) - base
        kf, cf, olo, ohi = got[:4]
        st["entries_out"] = kf.numel()
        st["ms"] = ms
        out = cls(k, kf, cf, olo, ohi, group, keys_lo_full=got[4] if two else None, path=path)
        out.stats["condition"] = st
        return out

    def close(self):
        if self.peer is not None:
            torch.cuda.synchronize()
            dist.barrier(self.group)              # nobody is still reading a peer's array
            self.peer.close(self.table.device)
            self.peer = None

    def scan(self, events=None):
        plot = self.scan_on(self.table, events)
        self._scanned = True
        return plot

    def scan_on(self, t, events=None):
        """one T_scan on table replica `t` (self.table for the resident scans, a freshly loaded
        replica in the e2e leg).  Peer mode keeps the phases ordered with two collectives per scan:
        a 4-byte all-reduce after pass 1 (every remote atomic has landed before any pass 2 reads),
        and the plot all-reduce after pass 2.  The incidence array is double-buffered: scan s uses
        buffer s&1 and clears the other one after the first barrier -- by then every rank has left
        pass 2 of scan s-1 (it could not have passed that scan's plot all-reduce otherwise), and
        nobody writes it before the plot all-reduce of scan s, which the clearing rank joins only
        after its memset (stream order)."""
        g = self.group
        self._scanned = False
        if self.path == "symm":
            return self._scan_symm(t, events)
        if self.peer is None:
            t.deg.zero_()
            t.plot.zero_()
            if events is not None:
                events[0].record()
            t.pass1()
            if events is not None:
                events[1].record()
            if self.world > 1:
                _in_place(lambda x: allreduce_deg(x, g), t.deg, g)
            t.pass2()
            if self.world > 1:
                _in_place(lambda x: allreduce_plot(x, g), t.plot, g)
            return t.plot
        par = self._step & 1
        self._step += 1
        t.deg_ptr = self.peer.own + par * self.peer.nbytes
        t.shards = self.peer.shards(self.offsets, par)
        if getattr(t, "_p2_scratch", None) is None:     # pass 2 batches its foreign look-ups through this
            t._p2_scratch = torch.empty(t.L.hm_pass2_scratch_bytes(t.hi - t.lo, t.idx64), dtype=torch.uint8,
                                        device=t.device)
        t.shards.scratch = t._p2_scratch.data_ptr()
        t.shards.scratch_bytes = t._p2_scratch.numel()
        ph = self._phase_events() if self.profile_phases else None
        t.plot.zero_()
        if events is not None:
            events[0].record()
        if ph: ph[0].record()
        t.pass1()
        if events is not None:
            events[1].record()
        if ph: ph[1].record()
        _in_place(lambda x: dist.all_reduce(x, group=g), self._barrier_t, g)   # all pass 1 kernels have landed
        if ph: ph[2].record()
        main = torch.cuda.current_stream()
        self._side.wait_stream(main)
        with torch.cuda.stream(self._side):                           # the next scan's buffer is cleared
            self._peer_views[par ^ 1].zero_()                         #   next to pass 2 ...
        t.pass2()
        if ph: ph[3].record()
        main.wait_stream(self._side)
        if ph: ph[4].record()
        _in_place(lambda x: allreduce_plot(x, g), t.plot, g)          # ... and before anybody can use it
        if ph: ph[5].record()
        return t.plot

    def _scan_symm(self, t, events=None):
        """strand-symmetric scan, sharded: run scan of the own (run-aligned) range -> all-gather of the
        Bloom segments -> resolve of the own candidates -> plot all-reduce.  No peer memory needed."""
        g = self.group
        ph = self._phase_events() if self.profile_phases else None
        t.plot.zero_()
        if events is not None:
            events[0].record()
        if ph: ph[0].record()
        t.runscan(mid_event=events[1] if events is not None else None)   # [0],[1]: the dominant kernel alone
        if ph: ph[1].record()
        if self.world > 1:
            _in_place(lambda x: exchange_segments(x, self.rank, g), t.bloom_view(), g)
        if ph: ph[2].record()
        t.resolve()
        if ph: ph[3].record(); ph[4].record()
        if self.world > 1:
            _in_place(lambda x: allreduce_plot(x, g), t.plot, g)
        if ph: ph[5].record()
        return t.plot

    def symm_ok(self) -> bool:
        """status words of the last symmetric scan on every rank (synchronises): all clean?"""
        bad = torch.zeros(1, dtype=torch.int32, device=self.table.device)
        if self.path == "symm":
            _, st = self.table.symm_status()
            bad[0] = int(st != 0)
        if self.world > 1:
            _in_place(lambda x: dist.all_reduce(x, op=dist.ReduceOp.MAX, group=self.group), bad, self.group)
        return int(bad.item()) == 0

    def extract(self, pixmap, dst: int = 0, timings: dict | None = None, budget: int | None = None):
        """extract_kmer_pairs' pair list for a pixel -> smudge map (uint16[SMAX+1, FMAX+1], label 0 = none): on rank
        `dst` the structured array hetmers.Scan.extract returns for the table, the same records in the same order;
        None on the other ranks.  Lists from the last scan() of the resident replica, or runs one first (its plot is
        dropped); stats["scan_reused"] says which.  Each rank lists its own range against its own replica:
          symm    the candidates of its run-aligned range (DeviceTable.extract); a dirty status word on any rank
                  raises on every rank;
          direct  its range of the direct passes' results (DeviceTable.pass2_extract), a count launch and then the
                  fill, reading the incidence bytes of the last scan (the peers' through PeerDeg, or the
                  all-reduced array in dense mode); a barrier at the end keeps the next scan_on from clearing an
                  incidence buffer a peer still reads.
        The records go through one device buffer of what `budget` (device bytes for the listing; default: free
        device memory minus _lib.BUDGET_RESERVE) leaves beside the pixmap and the counter: symm candidates in slices
        of half its records (at most two records each), direct entries in slices of its records (at most one each)
        when the count exceeds it.  Too little room for one slice is HM_ENOMEM on every rank, before any launch.
        The ranks' records are gathered on dst and sorted there (gather_pairs).
        timings (ms): scan, listing, d2h, gather_and_sort; stats: route, scan_reused, slices, records, ..."""
        lap = _lapper({} if timings is None else timings)
        with torch.cuda.device(self.table.device):
            recs = self._list_pairs(pixmap, lap, budget)
            t0 = time.perf_counter()
            res = gather_pairs(recs, dst, self.group)
            lap("gather_and_sort", t0)
        return res

    def _list_pairs(self, pixmap, lap, budget):
        """the listing of extract(): this rank's records (host, in the order listed); self.stats as extract() sets it.
        lap: the phases scan (when run), listing, d2h"""
        import numpy as np
        from . import _lib
        from .hetmers import PAIR_DTYPE
        g, t, dev = self.group, self.table, self.table.device
        pm = np.ascontiguousarray(pixmap, dtype=np.uint16).reshape(-1)
        if pm.size != _lib.PLOT_CELLS:
            raise ValueError(f"pixmap has {pm.size} cells, not {_lib.PLOT_CELLS}")
        item = PAIR_DTYPE.itemsize
        symm = self.path == "symm"
        with torch.cuda.device(dev):
            reused = self._scanned
            t0 = time.perf_counter()
            if not reused:                                      # (every rank has called the same methods)
                self.scan()
                torch.cuda.synchronize(dev)
                t0 = lap("scan", t0)
            if symm and not self.symm_ok():
                raise RuntimeError(f"rank {self.rank}: the last symmetric scan left a non-zero status word on some "
                                   f"rank; its candidates must not be listed")
            fixed = 2 * _lib.PLOT_CELLS + 256                   # the device pixmap and the record counter
            need = 2 if symm else 1                             # the records of one slice
            if budget is None:
                budget = torch.cuda.mem_get_info(dev)[0] - _lib.BUDGET_RESERVE
            room = max((budget - fixed) // item, 0)
            short = torch.tensor([int(room < need)], dtype=torch.int32, device=self._coll_dev)
            if self.world > 1:
                dist.all_reduce(short, op=dist.ReduceOp.MAX, group=g)
            if int(short.item()):
                raise _lib.HetmersError(-3, f"rank {self.rank}: listing k-mer pairs needs at least {fixed + need * item} "
                                            f"device bytes on every rank ({2 * _lib.PLOT_CELLS} for the pixmap, 256 for "
                                            f"the counter, {need} x {item} for one slice's records); the budget here is "
                                            f"{budget} bytes")
            d_pix = torch.from_numpy(pm.view(np.int16)).to(dev)
            count = torch.zeros(1, dtype=torch.int64, device=dev)
            if symm:
                nc, _ = t.symm_status()
                nc = min(nc, t.symm_layout.cand_cap)
                cap = max(min(room, 2 * nc), need)
                step = cap // 2
                ranges = [(c, min(c + step, nc)) for c in range(0, nc, step)]
            else:
                t.pass2_extract(d_pix, None, count)             # count launch
                total = int(count.item())
                cap = max(min(room, total), need)
                step = cap if total > cap else max(t.hi - t.lo, 1)
                ranges = [(a, min(a + step, t.hi)) for a in range(t.lo, t.hi, step)] if total else []
            out = torch.empty(cap * item, dtype=torch.uint8, device=dev)
            t0 = lap("listing", t0)
            parts = []
            for a, b in ranges:
                count.zero_()
                if symm:
                    t.extract(d_pix, out, count, a, b)
                else:
                    t.pass2_extract(d_pix, out, count, a, b)
                c = int(count.item())
                if c > cap:
                    raise _lib.HetmersError(-2, f"rank {self.rank}: {c} records listed from [{a}, {b}), beyond the "
                                                f"buffer of {cap}")
                t0 = lap("listing", t0)
                if c:
                    parts.append(out[:c * item].cpu().numpy())
                t0 = lap("d2h", t0)
            del out, d_pix, count
            recs = (np.concatenate(parts) if len(parts) > 1 else parts[0] if parts else
                    np.empty(0, dtype=np.uint8)).view(PAIR_DTYPE)
            if not symm and self.world > 1:                     # nobody clears what a peer still reads
                _in_place(lambda x: dist.all_reduce(x, group=g), self._barrier_t, g)
            self.stats = {"route": self.path, "scan_reused": reused, "slices": len(ranges), "records": len(recs),
                          "buffer_records": cap, "budget": budget, "range": [t.lo, t.hi],
                          **{key: v for key, v in self.stats.items() if key == "condition"}}
        return recs

    def write_pairs(self, sma, out, timings: dict | None = None, budget: int | None = None):
        """extract_kmer_pairs' output files for the smudges of `sma` (hetmers.read_sma): `<out>.<a>A<b>B.txt` per label,
        byte for byte what `extract_kmer_pairs -o<out> <table> <sma>` writes; every rank calls this.  The pairs are
        listed as extract() lists them (the same scan reuse, routes, refusals and stats), then the file phase
        (write_pair_files, DESIGN.md §6b) routes each record to the rank owning its key window, which sorts and formats
        them on its GPU and writes its segment of every file.  budget: device bytes per rank for the listing and for
        the file phase (default: free device memory minus _lib.BUDGET_RESERVE at each).  -> the file phase's stats,
        on every rank; timings (ms): the listing's phases, then hist_and_plan, route, all_to_all, sort, format,
        text_d2h, write"""
        pix, labels = read_sma_on_ranks(sma, self.group, self._coll_dev)
        lap = _lapper({} if timings is None else timings)
        with torch.cuda.device(self.table.device):
            recs = self._list_pairs(pix, lap, budget)
            return write_pair_files(recs, self.kmer, labels, out, self.group, self.table.device, budget, lap)

    profile_phases = False

    def _phase_events(self):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        self._phases = getattr(self, "_phases", [])
        self._phases.append(ev)
        return ev

    def phase_ms(self):
        """mean ms of (pass1, barrier, pass2, zero-next, plot all-reduce) over the profiled scans"""
        torch.cuda.synchronize()
        rows = [[a.elapsed_time(b) for a, b in zip(ev[:-1], ev[1:])] for ev in getattr(self, "_phases", [])]
        if not rows:
            return None
        names = ["pass1", "barrier_after_pass1", "pass2", "zero_next_buffer", "plot_allreduce"] if self.path != "symm" else \
                ["runscan", "bloom_allgather", "resolve", "-", "plot_allreduce"]
        return {n: sum(r[i] for r in rows) / len(rows) for i, n in enumerate(names)}

    # ---- end-to-end from pinned host buffers (bench.py e2e leg) -----------------------------
    def measure_e2e(self, steps, warmup):
        """per step: H2D of this rank's shard of raw FastK records + the stub index, unpack,
        shard exchange, bucket index, scan, plot D2H on rank 0.  -> e2e dict (max over ranks)."""
        from . import _lib
        from .device import DeviceTable
        t = self.table
        dev = t.device
        k, n, lo, hi = self.kmer, self.n_total, self.load_lo, self.load_hi
        wlo, whi = self.lo, self.hi
        kbyte, ibyte = (k + 3) // 4, 3
        pbyte = kbyte - ibyte + 2
        m = hi - lo
        keys, cnt = t.keys, t.cnt
        rec = torch.empty((m, pbyte), dtype=torch.uint8, device=dev)
        ks, cs = keys[lo:hi], cnt[lo:hi].to(torch.int32) & 0xFFFF
        for j in range(ibyte, kbyte):
            rec[:, j - ibyte] = ((ks >> (56 - 8 * j)) & 0xFF).to(torch.uint8)
        rec[:, pbyte - 2] = (cs & 0xFF).to(torch.uint8)
        rec[:, pbyte - 1] = ((cs >> 8) & 0xFF).to(torch.uint8)
        index = torch.cumsum(torch.bincount((keys >> 40) & 0xFFFFFF, minlength=1 << 24), 0)
        h_rec = torch.empty(rec.numel(), dtype=torch.uint8, pin_memory=True)
        h_rec.copy_(rec.view(-1))
        h_idx = torch.empty(1 << 24, dtype=torch.int64, pin_memory=True)
        h_idx.copy_(index)
        h_plot = torch.empty(_lib.PLOT_CELLS, dtype=torch.int64, pin_memory=True)
        del rec, index, ks, cs
        # the replica built by the timed call reuses no state of self.table
        d_rec = torch.empty(h_rec.numel(), dtype=torch.uint8, device=dev)
        d_idx = torch.empty(1 << 24, dtype=torch.int64, device=dev)
        k2 = torch.empty(n + self.world, dtype=torch.int64, device=dev)     # room for the all-gather's even chunks
        c2 = torch.empty(n + self.world, dtype=torch.int16, device=dev)

        def call():
            d_rec.copy_(h_rec, non_blocking=True)
            d_idx.copy_(h_idx, non_blocking=True)
            DeviceTable.from_records(k, ibyte, d_rec, d_idx, first=lo, out=(k2, c2))
            gather_table(k2[lo:hi], c2[lo:hi], self.group, out=(k2, c2))
            tt = DeviceTable(k, k2[:n], c2[:n], bits=self.bits).build_index(direct=(self.path != "symm"))
            if self.path == "symm":
                # (the fingerprint of the freshly unpacked shard is part of the timed call)
                if not fingerprint_verdict(tt.fingerprint(lo, hi, self.seeds), self.group):
                    raise RuntimeError("e2e replica is not symmetric although the resident table was")
                tt.alloc_symm(wlo, whi, self.table.symm_shards)
            else:
                tt.alloc_work(wlo, whi)
            self.scan_on(tt)
            if self.rank == 0:
                h_plot.copy_(tt.plot, non_blocking=True)
            torch.cuda.synchronize()
            return tt

        for _ in range(max(warmup, 1)):
            call()
        dist.barrier(self.group)
        t0 = time.perf_counter()
        for _ in range(steps):
            tt = call()
        dist.barrier(self.group)
        dt = torch.tensor([(time.perf_counter() - t0) / steps], dtype=torch.float64, device=dev)
        dist.all_reduce(dt, op=dist.ReduceOp.MAX, group=self.group)
        same = bool(torch.equal(tt.plot, t.plot)) if steps > 0 else True
        dtv = float(dt.item())
        h2d = torch.tensor([h_rec.numel() + h_idx.numel() * 8], dtype=torch.int64, device=dev)
        dist.all_reduce(h2d, group=self.group)                     # whole job, all ranks
        return {"value": n / dtv, "unit": "k-mers/s", "ms_per_step": dtv * 1e3,
                "h2d_bytes_per_step": int(h2d.item()),
                "d2h_bytes_per_step": int(_lib.PLOT_CELLS * 8),
                "api": "smudgeplot_b200.dist: pinned shard records -> H2D -> hm_k_unpack_records -> shard exchange "
                       "(NCCL) -> hm_k_build_bucket_index -> " +
                       ("fingerprint -> runscan -> all-gather(Bloom) -> resolve" if self.path == "symm" else
                        "filter -> pass1 -> deg exchange -> pass2") + " -> all-reduce(plot) -> D2H",
                "plot_matches_resident_scan": same, "exchange": self.exchange}


# ---- streaming a strand-symmetric table, each rank its own share (DESIGN.md §4c, *Ranks*) ------------------

def file_run_aligned_cuts(kt, world: int, window: int = 4096):
    """run_aligned_cuts of a FastK table (fastk.KtabFiles) from its files alone, the rule hm_rank_scan_create
    applies: c_r = the first run start at or after n*r/world, found by reading `window` records at a time after
    each nominal cut.  -> [0, c_1, ..., n]"""
    import numpy as np
    n, k = kt.nels, kt.kmer
    sh = np.uint64(64 - 2 * (k >> 1))
    part_end = np.cumsum(np.asarray(kt.part_nels, dtype=np.int64))

    def words(a, b):                       # word 0 of the keys of ordinals [a, b)
        out = np.zeros(b - a, dtype=np.uint64)
        pre = np.searchsorted(kt.index, np.arange(a, b, dtype=np.int64), side="right").astype(np.uint64)
        out |= pre << np.uint64(64 - 8 * kt.ibyte)
        for i in range(a, b):
            p = int(np.searchsorted(part_end, i, side="right"))
            j = i - (int(part_end[p - 1]) if p > 0 else 0)
            rec = kt.records[p][j * kt.pbyte:(j + 1) * kt.pbyte]
            for t in range(min(kt.hbyte, 8 - kt.ibyte)):
                out[i - a] |= np.uint64(int(rec[t])) << np.uint64(56 - 8 * (kt.ibyte + t))
        return out

    cuts = [0]
    for r in range(1, world):
        c = (n * r) // world
        if c <= cuts[-1]:
            cuts.append(cuts[-1])
            continue
        prev = words(c - 1, c)[0] >> sh
        at = n
        while c < n:
            w = words(c, min(n, c + window))
            d = np.nonzero((w >> sh) != prev)[0]
            if d.size:
                at = c + int(d[0])
                break
            c += w.size
        cuts.append(at)
    return cuts + [n]


# ---- trimming and symmetrising across the ranks (ShardedScan.from_ktab(L=...), DESIGN.md §4e) ---------------------

_U64 = (1 << 64) - 1


def share_range(n: int, world: int, rank: int):
    """the source ordinals rank `rank` of `world` loads: [n*rank/world, n*(rank+1)/world)"""
    return (n * rank) // world, (n * (rank + 1)) // world


def examine_window(n: int):
    """the ordinals whose counts decide "trimmed?" in hm_scan_examine: all of them when n + 3 < 1e8, else the 1e8
    around the middle -> (frst, last).  For n = 1e8 - 3 .. 1e8 - 1 that rule's window reaches 1 or 2 entries beyond
    the table at either end; here it is clipped to the table."""
    if n + 3 < 100_000_000:
        return 0, n
    return max(n // 2 - 50_000_000, 0), min(n // 2 + 50_000_000, n)


def condition_cuts(hist, world: int):
    """Cut the key prefixes into `world` contiguous ranges of near-equal output count, on prefix boundaries; hist:
    output entries per prefix (the same summed histogram on every rank, so every rank computes the same cuts).
    Cut r is the prefix boundary nearest to r/world of the total (the lower one on a tie), so a range is off its
    share by at most one prefix's count; ranges may be empty (one prefix may hold most of the table).
    -> [0, c_1, ..., c_{world-1}, len(hist)], rank d owning prefixes [c_d, c_{d+1})"""
    import numpy as np
    h = np.asarray(hist, dtype=np.int64)
    np_ = h.size
    before = np.zeros(np_ + 1, dtype=np.int64)                 # before[p]: entries under prefixes below p
    np.cumsum(h, out=before[1:])
    total = int(before[-1])
    cuts = [0]
    for r in range(1, world):
        want = (total * r) // world
        p = int(np.searchsorted(before, want, side="right")) - 1
        if p < np_ and before[p + 1] - want < want - before[p]:
            p += 1
        cuts.append(max(p, cuts[-1]))
    return cuts + [np_]


def _signed(v: int) -> int:
    return v - (1 << 64) if v >= (1 << 63) else v


def _revcomp_words(x0: int, x1: int, k: int):
    """reverse complement of a left-aligned packed k-mer (unsigned words; x1: bases 32.. for k > 32) -> (w0, w1)"""
    bits = 128 if k > 32 else 64
    v = ((x0 << 64) | x1 if k > 32 else x0) >> (bits - 2 * k)
    r = 0
    for _ in range(k):
        r = (r << 2) | (3 - (v & 3))
        v >>= 2
    r <<= bits - 2 * k
    return (r >> 64, r & _U64) if k > 32 else (r, 0)


def _u64_bounds(keys: torch.Tensor, q: int, lo: int, hi: int):
    """[a, b): the entries of keys[lo:hi] equal to the unsigned value q.  keys are sorted as unsigned numbers but
    held as int64, which torch compares signed: the entries below 2^63 come first, then those at or above (negative
    as int64), each part sorted in signed order too; q is searched in its part"""
    a, b = lo, hi
    while a < b:                                               # the first entry at or above 2^63
        mid = (a + b) // 2
        if int(keys[mid]) >= 0:
            a = mid + 1
        else:
            b = mid
    qs = _signed(q)
    p0, p1 = (lo, a) if qs >= 0 else (a, hi)
    if p0 >= p1:
        return p0, p0
    part, v = keys[p0:p1], torch.tensor([qs], dtype=torch.int64, device=keys.device)
    return p0 + int(torch.searchsorted(part, v)), p0 + int(torch.searchsorted(part, v, right=True))


def _share_find(keys: torch.Tensor, keys_lo, q0: int, q1: int) -> int:
    """index of the k-mer (q0, q1) in a sorted share (keys_lo: second words, k > 32), or -1"""
    a, b = _u64_bounds(keys, q0, 0, keys.numel())
    if keys_lo is not None and a < b:
        a, b = _u64_bounds(keys_lo, q1, a, b)
    return a if a < b else -1


def job_examine(ethresh: int, kmer: int, n: int, keys: torch.Tensor, keys_lo, min_count, group=None,
                coll_dev=None):
    """hm_scan_examine's decisions on a table of n entries whose ranks hold the shares of share_range: keys /
    keys_lo (k > 32) this rank's sorted share; min_count(a, b) the smallest count >= 1 (read as int16) among its
    entries [a, b), 0x8000 if none.  trim: the MIN over the ranks of min_count over their parts of examine_window(n)
    is >= ethresh.  symm: from sidx = 1, the owner of entry sidx broadcasts the reverse complement of its key, every
    rank looks it up in its share, and a MAX all-reduce gives its position or -1: -1 = not symmetric, another
    position = symmetric, sidx itself (a palindrome) = go on with sidx + 1; n <= 1 counts as symmetric.
    -> (trimmed?, symmetric?) on every rank"""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    lo, hi = share_range(n, world, rank)
    frst, last = examine_window(n)
    a, b = max(lo, frst), min(hi, last)
    low = torch.tensor([min_count(a - lo, b - lo) if a < b else 0x8000], dtype=torch.int64, device=coll_dev)
    dist.all_reduce(low, op=dist.ReduceOp.MIN, group=group)
    trimmed = int(low.item()) >= ethresh
    symmetric = True
    owner = lambda i: next(r for r in range(world) if share_range(n, world, r)[1] > i)   # noqa: E731
    sidx = 1
    while sidx < n:
        src = owner(sidx)
        q = torch.zeros(2, dtype=torch.int64, device=coll_dev)
        if rank == src:
            x1 = int(keys_lo[sidx - lo]) & _U64 if keys_lo is not None else 0
            r0, r1 = _revcomp_words(int(keys[sidx - lo]) & _U64, x1, kmer)
            q[0], q[1] = _signed(r0), _signed(r1)
        dist.broadcast(q, src=dist.get_global_rank(group, src) if group is not None else src, group=group)
        i = _share_find(keys, keys_lo, int(q[0]) & _U64, int(q[1]) & _U64)
        pos = torch.tensor([lo + i if i >= 0 else -1], dtype=torch.int64, device=coll_dev)
        dist.all_reduce(pos, op=dist.ReduceOp.MAX, group=group)
        p = int(pos.item())
        if p < 0:
            symmetric = False
            break
        if p != sidx:
            break
        sidx += 1
    return trimmed, symmetric


def _condition_share(k, ibyte, m, share, ethr, do_symm, budget, group, coll, st, done, t):
    """the conditioning steps of ShardedScan._from_ktab_conditioned on this rank's source share (share: [keys,
    counts, second words or None] of m entries, emptied here so that the share is freed as soon as it has been
    routed, or refused) -> this rank's conditioned share (keys, counts, second words or None)"""
    import ctypes as C
    import numpy as np
    from . import _lib
    from .device import _ptr, _stream
    Lb = _lib.lib()
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    sk, sc, sl = share
    share.clear()
    dev, two = sk.device, k > 32
    # histograms of this share: kept originals, and kept originals + reverse complements, per key prefix
    hist = torch.zeros((2, 1 << min(_lib.COND_HIST_BITS, 2 * k)), dtype=torch.int64, device=dev)
    for row, symm in ((0, 0), (1, do_symm)):
        _lib.check(Lb.hm_k_cond_hist(_ptr(sk), _ptr(sl), _ptr(sc), m, k, ethr, symm, _ptr(hist[row]), _stream()))
    sent = int(hist[1].sum())
    _in_place(lambda x: dist.all_reduce(x, group=group), hist, group)
    h = hist.cpu().numpy()
    del hist
    cuts = condition_cuts(h[1], world)
    at_all = np.concatenate([[0], np.cumsum(h[1])])[cuts]
    at_orig = np.concatenate([[0], np.cumsum(h[0])])[cuts]
    recv = np.diff(at_all).tolist()
    recv_rc = (np.diff(at_all) - np.diff(at_orig)).tolist()
    total_orig, total = int(h[0].sum()), int(h[1].sum())
    need = Lb.hm_shard_condition_bytes(k, ibyte, world, m, sent, recv[rank], recv_rc[rank], total, int(do_symm))
    sizes = torch.zeros((world, 2), dtype=torch.int64, device=coll)
    sizes[rank, 0], sizes[rank, 1] = need, budget
    dist.all_reduce(sizes, group=group)
    needs, budgets = sizes[:, 0].tolist(), sizes[:, 1].tolist()
    st.update(working_set_bytes=need, prefix_cuts=cuts)
    big = [d for d in range(world) if two and do_symm and recv_rc[d] >= 0xFFFFFFF0]
    short = [d for d in range(world) if needs[d] > budgets[d]]
    if big or short:
        del sk, sc, sl
        if big:
            raise _lib.HetmersError(-6, f"rank {rank}: conditioning across {world} ranks would send ranks {big} "
                                        f"{[recv_rc[d] for d in big]} reverse complements of k={k} to sort: 2^32 - 16 "
                                        f"or more needs 64-bit sort indices")
        raise _lib.HetmersError(-3, f"rank {rank}: conditioning across {world} ranks needs {needs} device bytes per "
                                    f"rank, beyond the budgets {budgets} of ranks {short}")
    t = done("hist_and_plan", t)
    share = [sk, sc, sl]
    del sk, sc, sl
    dest = np.repeat(np.arange(world, dtype=np.int16), np.diff(cuts))
    out, sent_to, got_from = _route_exchange_settle(k, m, share, ethr, do_symm, torch.from_numpy(dest).to(dev), False,
                                                    (sent, recv[rank], recv_rc[rank], total_orig, total - total_orig),
                                                    group, coll, done, t)
    st.update(sent=sent_to, received=got_from)
    return out


def _route_exchange_settle(k, m, share, ethr, do_symm, dest, window, expect, group, coll, done, t):
    """One pass of conditioning across the ranks: every kept entry of this rank's source share (share: [keys, counts,
    second words or None] of m entries) and its reverse complement are routed to the rank owning its key prefix
    (dest: int16 per prefix; with window, -1 marks a prefix outside this pass), the two regions are all-to-all'ed,
    and the received entries are settled when symmetrising.  Without window the share list is emptied once routed,
    so that its entries are freed before the exchange.  expect: (entries sent, received, reverse complements
    received, and over all ranks kept originals and reverse complements routed) as the histograms count them.
    done(phase, t): the phases "route", "exchange", "sort_and_merge".
    -> ((keys, counts, second words or None) of the settled entries, entries sent to each rank, received from each)"""
    import ctypes as C
    import numpy as np
    from . import _lib
    from .device import _ptr, _stream
    Lb = _lib.lib()
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    sk, sc, sl = share
    if not window:
        share.clear()
    dev, two = sk.device, k > 32
    route_count = Lb.hm_k_shard_route_count_window if window else Lb.hm_k_shard_route_count
    route_scatter = Lb.hm_k_shard_route_scatter_window if window else Lb.hm_k_shard_route_scatter

    # route: every kept entry (and its reverse complement) to the rank owning its key prefix
    counts = torch.zeros(2 * world + 2, dtype=torch.int64, device=dev)
    tiles = torch.empty(m // 256 + 2, dtype=torch.int64, device=dev)
    _lib.check(route_count(_ptr(sk), _ptr(sl), _ptr(sc), m, k, ethr, int(do_symm), _ptr(dest), world, _ptr(counts),
                           _ptr(tiles), _stream()))
    c = counts.tolist()
    so, sr = c[:world], c[world:2 * world]
    n_o, n_r = sum(so), sum(sr)
    assert n_o + n_r == expect[0] and c[2 * world] == n_o, (so, sr, expect, c[2 * world])
    send_k = torch.empty(max(n_o + n_r, 1), dtype=torch.int64, device=dev)
    send_c = torch.empty(max(n_o + n_r, 1), dtype=torch.int16, device=dev)
    send_l = torch.empty(max(n_o + n_r, 1), dtype=torch.int64, device=dev) if two else None
    cursor = torch.tensor(np.concatenate([[0], np.cumsum(sr)[:-1]]).astype(np.int64), device=dev)
    _lib.check(route_scatter(_ptr(sk), _ptr(sl), _ptr(sc), m, k, ethr, int(do_symm), _ptr(dest), _ptr(tiles),
                             _ptr(send_k), _ptr(send_l), _ptr(send_c), n_o, n_r, _ptr(cursor),
                             _ptr(counts[2 * world + 1:]), _stream()))
    del sk, sc, sl, tiles, dest, cursor
    flag = counts[2 * world + 1:].to(coll)
    dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=group)
    if int(flag.item()):
        raise _lib.HetmersError(-2, f"rank {rank}: routing the conditioned entries overran the send buffer on a rank")
    t = done("route", t)

    # exchange: the originals' region and the reverse complements' region, each all-to-all'ed
    mine = torch.tensor([so, sr], dtype=torch.int64).t().contiguous().to(coll)
    theirs = torch.empty_like(mine)
    dist.all_to_all_single(theirs, mine, group=group)
    ro, rr = theirs[:, 0].tolist(), theirs[:, 1].tolist()
    r_o, r_c = sum(ro), sum(rr)
    assert r_o + r_c == expect[1] and r_c == expect[2], (ro, rr, expect)
    room = max(r_o + r_c, 1)
    rk = torch.empty(room, dtype=torch.int64, device=dev)
    rc = torch.empty(room, dtype=torch.int16, device=dev)
    rl = torch.empty(room, dtype=torch.int64, device=dev) if two else None
    for (a, b, c0, c1, ins, outs, job_total) in ((0, r_o, 0, n_o, so, ro, expect[3]),
                                                 (r_o, r_o + r_c, n_o, n_o + n_r, sr, rr, expect[4])):
        if job_total == 0:
            continue
        _all_to_all(rk[a:b], send_k[c0:c1], outs, ins, group)
        if two:
            _all_to_all(rl[a:b], send_l[c0:c1], outs, ins, group)
        _all_to_all(rc[a:b].view(torch.uint8), send_c[c0:c1].view(torch.uint8), [2 * x for x in outs],
                    [2 * x for x in ins], group)
    del send_k, send_c, send_l
    t = done("exchange", t)
    sent_to, got_from = [a + b for a, b in zip(so, sr)], [a + b for a, b in zip(ro, rr)]
    if not do_symm:                                            # the originals arrive sorted: nothing to settle
        return (rk[:r_o], rc[:r_o], rl[:r_o] if two else None), sent_to, got_from

    # settle: sort the received reverse complements, merge them with the originals
    ok, oc = torch.empty(room, dtype=torch.int64, device=dev), torch.empty(room, dtype=torch.int16, device=dev)
    ol = torch.empty(room, dtype=torch.int64, device=dev) if two else None
    scratch = torch.empty(Lb.hm_k_shard_settle_bytes(k, r_o + r_c, r_c), dtype=torch.uint8, device=dev)
    n_out = C.c_int64()
    _lib.check(Lb.hm_k_shard_settle(k, _ptr(rk), _ptr(rl), _ptr(rc), r_o, r_c, _ptr(scratch), scratch.numel(),
                                    _ptr(ok), _ptr(ol), _ptr(oc), C.byref(n_out), _stream()))
    del rk, rc, rl, scratch
    done("sort_and_merge", t)
    e = n_out.value
    return (ok[:e], oc[:e], ol[:e] if two else None), sent_to, got_from


# ---- trimming and symmetrising across the ranks into new table files (condition_ktab, DESIGN.md §4f) --------------

def bucket_condition_cuts(hist, world: int, hb: int, ibyte: int):
    """condition_cuts on stub-index bucket boundaries, so that every rank's part of the table starts on a bucket
    (the reference bisects a table on disk by its buckets).  hist: output entries per hb-bit key prefix; a bucket
    holds the first 8*ibyte bits.  Where buckets are coarser than prefixes (8*ibyte < hb) the cut is made over the
    histogram summed per bucket and scaled back to prefixes.  -> [0, c_1, ..., c_{world-1}, 2^hb]"""
    return _coarse_condition_cuts(hist, world, hb, 8 * ibyte)


def run_condition_cuts(hist, world: int, hb: int, ibyte: int, kmer: int):
    """bucket_condition_cuts coarsened to run boundaries, so that every rank's part of the table starts on a run (the
    entries sharing their first kmer//2 bases) as pass 1 of the streamed scan needs: cuts on prefixes of min(hb,
    8*ibyte, 2*(kmer//2)) bits, made over the histogram summed per such prefix.  Where runs are no finer than
    buckets (2*(kmer//2) >= 8*ibyte) these are bucket_condition_cuts.  -> [0, c_1, ..., c_{world-1}, 2^hb]"""
    return _coarse_condition_cuts(hist, world, hb, min(8 * ibyte, 2 * (kmer >> 1)))


def _coarse_condition_cuts(hist, world: int, hb: int, bits: int):
    """condition_cuts on the boundaries of `bits`-bit key prefixes, hist counting per hb-bit prefix"""
    import numpy as np
    sh = hb - bits
    if sh <= 0:
        return condition_cuts(hist, world)
    h = np.asarray(hist, dtype=np.int64).reshape(-1, 1 << sh).sum(axis=1)
    return [c << sh for c in condition_cuts(h, world)]


def prefix_buckets(p0: int, p1: int, hb: int, ibyte: int):
    """the stub buckets [b0, b1) that hold the keys of the hb-bit prefixes [p0, p1), p0 < p1"""
    b = 8 * ibyte
    if b >= hb:
        return p0 << (b - hb), p1 << (b - hb)
    return p0 >> (hb - b), ((p1 - 1) >> (hb - b)) + 1


def rank_sub_cuts(kmer: int, ibyte: int, shares, do_symm, budgets, hist, cuts):
    """every rank's range of key prefixes [cuts[d], cuts[d+1]) cut into the sub-ranges its budget allows beside its
    resident share (hm_rank_condition_cut; shares[d]: rank d's source entries, budgets[d]: its device bytes, hist:
    output entries per prefix summed over the ranks) -> per rank [cuts[d], ..., cuts[d+1]], the bounds of its
    sub-ranges.  HM_ENOMEM naming the rank and the sizes when one prefix, or the load, does not fit."""
    import ctypes as C
    import numpy as np
    from . import _lib
    Lb = _lib.lib()
    world = len(shares)
    h = np.ascontiguousarray(hist, dtype=np.int64)
    out = []
    for d in range(world):
        a, b = int(cuts[d]), int(cuts[d + 1])
        seg = np.ascontiguousarray(h[a:b])
        sub = np.zeros(b - a + 1, dtype=np.int64)
        n_sub = C.c_int64()
        rc = Lb.hm_rank_condition_cut(kmer, ibyte, world, int(shares[d]), int(do_symm), int(budgets[d]),
                                      seg.ctypes.data, b - a, sub.ctypes.data, C.byref(n_sub))
        if rc != 0:
            raise _lib.HetmersError(rc, f"rank {d}: " + Lb.hm_last_error().decode(errors="replace"))
        out.append((sub[:n_sub.value + 1] + a).tolist())
    return out


def rank_pass_counts(h_local, h_all, subs, rank: int):
    """what the histograms say of each pass before any entry moves: pass p routes the p-th sub-range of every rank
    that has one (subs: rank_sub_cuts).  h_local / h_all: [kept originals, kept originals + reverse complements] per
    prefix of this rank's share / summed over the ranks.  -> per pass (entries this rank sends, entries it
    receives, reverse complements among them, kept originals routed by all ranks, reverse complements routed)"""
    import numpy as np

    def cum(row):
        return np.concatenate([[0], np.cumsum(np.asarray(row, dtype=np.int64))])
    s_loc, a_orig, a_all = cum(h_local[1]), cum(h_all[0]), cum(h_all[1])
    out = []
    for p in range(max(len(s) - 1 for s in subs)):
        win = [(s[p], s[p + 1]) for s in subs if p < len(s) - 1]
        sent = sum(int(s_loc[b] - s_loc[a]) for a, b in win)
        orig = sum(int(a_orig[b] - a_orig[a]) for a, b in win)
        every = sum(int(a_all[b] - a_all[a]) for a, b in win)
        if p < len(subs[rank]) - 1:
            a, b = subs[rank][p], subs[rank][p + 1]
            recv, rc = int(a_all[b] - a_all[a]), int((a_all[b] - a_all[a]) - (a_orig[b] - a_orig[a]))
        else:
            recv = rc = 0
        out.append((sent, recv, rc, orig, every - orig))
    return out


def raise_on_any_rank(err, what: str, coll, group=None):
    """One flag all-reduce where a rank may have failed (a rank's lists in host memory: StreamedShardedScan with a
    list_host_budget).  err: this rank's HetmersError, or None -> returns if no rank failed; else raises on every
    rank: this rank's own error, or a HetmersError with the failing rank's code naming the ranks that failed, so
    that no rank is left waiting in the next collective."""
    from . import _lib
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    codes = _reduce([int(err.code) if err is not None and d == rank else 0 for d in range(world)], coll, group)
    bad = [d for d, c in enumerate(codes) if c]
    if not bad:
        return
    if err is not None:
        raise err
    raise _lib.HetmersError(codes[bad[0]], f"rank {rank}: {what} failed on rank{'s' if len(bad) > 1 else ''} "
                                           f"{', '.join(map(str, bad))} (codes {[codes[d] for d in bad]})")


def pass1_agreement(fp, spilled: bool, err, coll, group=None):
    """The job-wide verdicts after pass 1 of ranks that may keep their lists in host memory, in one all-gather:
    fp = this rank's four fingerprint sums (uint64), spilled = its lists went to host memory, err = its
    HetmersError or None.  -> (symmetric, spilled on any rank); a rank's failure raises on every rank, as
    raise_on_any_rank does."""
    from . import _lib
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    mine = torch.tensor([_signed(int(v)) for v in fp] + [int(bool(spilled) and err is None),
                                                        int(err.code) if err is not None else 0],
                        dtype=torch.int64, device=coll)
    parts = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(parts, mine, group=group)
    rows = [p.tolist() for p in parts]
    bad = [d for d, r in enumerate(rows) if r[5]]
    if bad:
        if err is not None:
            raise err
        raise _lib.HetmersError(rows[bad[0]][5], f"rank {rank}: pass 1 failed on rank{'s' if len(bad) > 1 else ''} "
                                                 f"{', '.join(map(str, bad))} (codes {[rows[d][5] for d in bad]})")
    tot = [sum(r[i] for r in rows) & _U64 for i in range(4)]
    return tot[0] == tot[2] and tot[1] == tot[3], any(r[4] for r in rows)


def _reduce(vals, coll, group, op=dist.ReduceOp.SUM):
    """all_reduce of a list of integers -> the reduced list"""
    x = torch.tensor(vals, dtype=torch.int64, device=coll)
    dist.all_reduce(x, op=op, group=group)
    return x.tolist()


def _write_atomic(path: str, data: bytes):
    """write `data` as the file `path`: under a temporary name in its directory, then renamed into place"""
    import tempfile
    fd, tmp = tempfile.mkstemp(prefix="." + os.path.basename(path) + ".", suffix=".tmp", dir=os.path.dirname(path))
    try:
        with os.fdopen(fd, "wb") as f:
            f.write(data)
        os.rename(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise


class _RankConditioning:
    """One rank's part of trimming and symmetrising the FastK table kt across the ranks (condition_ktab,
    StreamedShardedScan.from_ktab).  The constructor loads the rank's share of the source onto dev and takes
    hetmers' decisions on the whole table (job_examine); needed() tells whether a step is.  plan() cuts the key
    prefixes into the ranks' ranges (cut_rule(hist, world, hb)) and every range into the passes its
    budget allows beside the resident share; run(take) conditions them, handing each pass's packed records to
    take.  close() frees the share.  st: the stats both callers report; ms: ms per phase."""

    def __init__(self, kt, ethresh, group, dev, coll, budget, ms):
        from . import _lib
        from .device import _ptr, _stream
        self.group, self.dev, self.coll, self.budget, self.ms = group, dev, coll, budget, ms
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.lap = _lapper(ms)
        self.k, self.n, self.ibyte, self.ethresh = kt.kmer, kt.nels, kt.ibyte, ethresh
        t = time.perf_counter()
        lo, hi = share_range(self.n, self.world, self.rank)
        self.m = hi - lo
        self.share = list(_load_share(kt, lo, hi, dev))
        t = self.done("load", t)
        Lb, share = _lib.lib(), self.share

        def share_min(a, b):
            out = torch.full((1,), 0x8000, dtype=torch.int32, device=dev)
            _lib.check(Lb.hm_k_min_count(_ptr(share[1]), a, b, _ptr(out), _stream()))
            return int(out.item())

        self.trimmed, self.symmetric = job_examine(ethresh, self.k, self.n, share[0], share[2], share_min, group,
                                                   coll)
        self.do_trim, self.do_symm = not self.trimmed, not self.symmetric
        self.lap("examine", t)
        self.st = {"trimmed": self.trimmed, "symmetric": self.symmetric,
                   "steps": (["trim"] if self.do_trim else []) + (["symmetrise"] if self.do_symm else []),
                   "entries_in": self.n}

    def done(self, phase, t):                              # the phase's kernels have finished
        torch.cuda.synchronize(self.dev)
        return self.lap(phase, t)

    def needed(self) -> bool:
        return self.do_trim or self.do_symm

    def close(self):
        self.share.clear()

    def plan(self, cut_rule, what: str):
        """histograms, the rank cuts, every rank's sub-ranges and every pass's counts.  HM_ENOMEM on every rank
        (the share freed) when a rank's share and one pass do not fit its budget; what: the job, for the message"""
        import numpy as np
        from . import _lib
        from .device import _ptr, _stream
        Lb, k, world, rank, share = _lib.lib(), self.k, self.world, self.rank, self.share
        t = time.perf_counter()
        self.ethr = self.ethresh if self.do_trim else 0
        self.hb = hb = min(_lib.COND_HIST_BITS, 2 * k)
        hist = torch.zeros((2, 1 << hb), dtype=torch.int64, device=self.dev)
        for row, symm in ((0, 0), (1, self.do_symm)):
            _lib.check(Lb.hm_k_cond_hist(_ptr(share[0]), _ptr(share[2]), _ptr(share[1]), self.m, k, self.ethr, symm,
                                         _ptr(hist[row]), _stream()))
        h_loc = hist.cpu().numpy()
        _in_place(lambda x: dist.all_reduce(x, group=self.group), hist, self.group)
        self.h_all = h_all = hist.cpu().numpy()
        del hist
        self.cuts = cuts = cut_rule(h_all[1], world, hb)
        budgets = _reduce([self.budget if d == rank else 0 for d in range(world)], self.coll, self.group)
        shares = [b - a for a, b in (share_range(self.n, world, d) for d in range(world))]
        try:
            self.subs = subs = rank_sub_cuts(k, self.ibyte, shares, self.do_symm, budgets, h_all[1], cuts)
        except _lib.HetmersError:
            self.close()
            raise
        self.passes = rank_pass_counts(h_loc, h_all, subs, rank)
        need = max(Lb.hm_rank_condition_bytes(k, self.ibyte, world, self.m, *c[:3], int(self.do_symm))
                   for c in self.passes)
        needs = _reduce([need if d == rank else 0 for d in range(world)], self.coll, self.group)
        short = [d for d in range(world) if needs[d] > budgets[d]]
        if short:
            self.close()
            raise _lib.HetmersError(-3, f"rank {rank}: conditioning {what} across {world} ranks needs {needs} "
                                        f"device bytes per rank, beyond the budgets {budgets} of ranks {short}; use "
                                        f"more ranks, or condition_kmer_table")
        self.span = prefix_buckets(cuts[rank], cuts[rank + 1], hb, self.ibyte) if cuts[rank] < cuts[rank + 1] \
            else (0, 0)
        self.bcounts = np.zeros(self.span[1] - self.span[0], dtype=np.int64)
        self.st.update(passes=len(self.passes), prefix_cuts=cuts, sub_ranges=subs[rank], sent=[], received=[],
                       budget=self.budget, working_set_bytes=need)
        self.done("hist_and_plan", t)

    def rank_entries(self, d: int) -> int:
        """the conditioned entries rank d receives, from the summed histogram"""
        a, b = self.cuts[d], self.cuts[d + 1]
        return int(self.h_all[1][a:b].sum())

    def run(self, take):
        """the passes: this rank's sub-range p conditioned and packed (its records' stub-bucket counts added to
        self.bcounts over self.span), then take(records, keys) with the pass's device records (uint8, in key
        order) and keys (their first words, int64); take must not keep either.  The share is freed at the end."""
        import numpy as np
        from . import _lib
        from .device import _ptr, _stream
        Lb, k, ibyte, hb, world, rank = _lib.lib(), self.k, self.ibyte, self.hb, self.world, self.rank
        pbyte = ((k + 3) >> 2) - ibyte + 2
        subs, span = self.subs, self.span
        self.ms["passes"] = []
        for p, expect in enumerate(self.passes):
            pm = {}
            self.ms["passes"].append(pm)
            plap = _lapper(pm)

            def pdone(phase, t0):
                torch.cuda.synchronize(self.dev)
                return plap("settle" if phase == "sort_and_merge" else phase, t0)
            dest = np.full(1 << hb, -1, dtype=np.int16)
            for d in range(world):
                if p < len(subs[d]) - 1:
                    dest[subs[d][p]:subs[d][p + 1]] = d
            (ok, oc, ol), sent_to, got_from = _route_exchange_settle(
                k, self.m, self.share, self.ethr, self.do_symm, torch.from_numpy(dest).to(self.dev), True, expect,
                self.group, self.coll, pdone, time.perf_counter())
            self.st["sent"].append(sum(sent_to))
            self.st["received"].append(sum(got_from))
            t = time.perf_counter()
            e = ok.numel()
            if e:
                b0, b1 = prefix_buckets(subs[rank][p], subs[rank][p + 1], hb, ibyte)
                rec = torch.empty(e * pbyte, dtype=torch.uint8, device=self.dev)
                bc = torch.empty(b1 - b0, dtype=torch.int64, device=self.dev)
                _lib.check(Lb.hm_k_cond_pack(k, ibyte, _ptr(ok), _ptr(ol), _ptr(oc), e, b0, b1 - b0, _ptr(rec),
                                             _ptr(bc), _stream()))
                self.bcounts[b0 - span[0]:b1 - span[0]] += bc.cpu().numpy()
                del bc
                take(rec, ok)
                del rec
            del ok, oc, ol
            pdone("pack", t)
        self.close()


def condition_ktab(src, dst, L, group=None, device=None, budget=None):
    """Trim and / or symmetrise the FastK table `src` into the new FastK table `dst` across the ranks of the group,
    every rank calling this (DESIGN.md §4f).  hetmers' decisions are taken on the whole table as from_ktab(L=...)
    takes them (job_examine): a table that needs neither step gives None on every rank and nothing is written.
    Otherwise `dst` holds, entry for entry, what hetmers.condition_table(src, dst, L) writes: the kept entries
    (count >= L when trimming) and, when symmetrising, their reverse complements with the same count, the original
    winning over an equal reverse complement; the same kmer and ibyte; minval max(source minval, L) when trimmed.

    Rank d owns one contiguous range of key prefixes, cut on stub-bucket boundaries, and writes its part
    `.<root>.ktab.<p>`, p counting the ranks with a non-empty output up to d (a rank with none writes no part);
    rank 0 writes the stub last.  Each rank loads its share of the source once and keeps it on the device while its
    range is conditioned in passes, a sub-range per pass, sized to `budget` (device bytes per rank; default: free
    memory minus _lib.BUDGET_RESERVE).  Refused on every rank before anything is written: a `dst` naming `src`
    (HM_EINVAL), a rank whose share and one pass do not fit its budget (HM_ENOMEM, with the sizes).  A failure to
    write on any rank raises on every rank and leaves no file under dst's names and no temporary file.  Returns on
    every rank once the files are in place.  -> stats of this rank: verdicts, steps, entries in / out (the job's
    and this rank's), passes, the prefix cuts and sub-ranges, entries sent / received per pass, part number and
    part count, bytes written, peak device bytes (torch's allocator; its peak statistics are reset) against the
    planned working set and the budget, and ms per phase (per pass: route, exchange, settle, pack)"""
    import concurrent.futures as cf
    import struct
    import tempfile
    import numpy as np
    from . import _lib, fastk
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    dev = torch.device(device if device is not None else "cuda")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    coll = dev if _nccl(group) else torch.device("cpu")
    ethresh = int(L)
    src, dst = str(src), str(dst)
    ms = {}
    lap = _lapper(ms)

    with torch.cuda.device(dev):
        if budget is None:
            budget = torch.cuda.mem_get_info(dev)[0] - _lib.BUDGET_RESERVE
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        kt = fastk.read_ktab(src, mmap=True)
        k, ibyte, src_parts = kt.kmer, kt.ibyte, kt.nparts
        if max(_reduce([int(fastk.same_table_files(src, src_parts, dst))], coll, group, dist.ReduceOp.MAX)):
            raise _lib.HetmersError(-1, f"rank {rank}: {dst} names the source table: conditioning writes a new table")
        minval_src = kt.minval
        job = _RankConditioning(kt, ethresh, group, dev, coll, budget, ms)
        del kt
        if not job.needed():
            job.close()
            return None
        do_trim = job.do_trim
        job.plan(lambda h, w, hb: bucket_condition_cuts(h, w, hb, ibyte), f"{src} into files")

        # the passes: this rank's sub-range p conditioned, packed and appended to its temporary part
        ddir, root = fastk.split_name(dst)
        pbyte = ((k + 3) >> 2) - ibyte + 2
        span, bcounts = job.span, job.bcounts
        fd, tmp, err = -1, "", None
        try:
            fd, tmp = tempfile.mkstemp(prefix=f".{root}.ktab.", suffix=f".rank{rank}.tmp", dir=ddir)
        except OSError as x:
            err = f"{ddir}: {x}"
        if max(_reduce([int(err is not None)], coll, group, dist.ReduceOp.MAX)):
            job.close()
            if fd >= 0:
                os.close(fd)
                os.unlink(tmp)
            raise _lib.HetmersError(-4, f"rank {rank}: cannot write {dst} on every rank" + (f": {err}" if err else ""))
        busy = [0.0]

        def append(buf):                                   # the writer thread (os.write releases the GIL)
            t0 = time.perf_counter()
            mv = memoryview(buf)
            while len(mv):
                mv = mv[os.write(fd, mv):]
            busy[0] += (time.perf_counter() - t0) * 1e3

        writer = cf.ThreadPoolExecutor(1)
        pending, n_out, part, nparts, total = None, 0, None, 0, 0
        st = job.st

        def take(rec, keys):
            nonlocal pending, err, n_out
            host = rec.cpu().numpy()
            if pending is not None and err is None:        # the last pass's records have been written
                try:
                    pending.result()
                except OSError as x:
                    err = f"{tmp}: {x}"
            if err is None:
                pending = writer.submit(append, host)
            n_out += keys.numel()

        try:
            os.write(fd, struct.pack("<iq", k, 0))         # the count is set once every pass is written
            job.run(take)
            t = time.perf_counter()
            if pending is not None and err is None:
                try:
                    pending.result()
                except OSError as x:
                    err = f"{tmp}: {x}"
            writer.shutdown(wait=True)
            if err is None:
                try:
                    os.pwrite(fd, struct.pack("<q", n_out), 4)
                except OSError as x:
                    err = f"{tmp}: {x}"
            os.close(fd)
            fd = -1

            # commit: every rank's part renamed into place once all succeeded, then the stub from rank 0
            got = _reduce(sum(([n_out, int(err is not None)] if d == rank else [0, 0] for d in range(world)), []),
                          coll, group)
            outs, failed = got[0::2], [d for d in range(world) if got[2 * d + 1]]
            if failed:
                raise _lib.HetmersError(-4, f"rank {rank}: writing {dst} failed on ranks {failed}"
                                            + (f": {err}" if err else ""))
            total = sum(outs)
            nparts = sum(1 for x in outs if x > 0)
            old_parts = 0
            if rank == 0 and os.path.exists(fastk.stub_path(dst)):
                with open(fastk.stub_path(dst), "rb") as f:
                    old_parts = max(struct.unpack("<4i", f.read(16))[1], 0)
            bad = None
            if n_out > 0:
                part = sum(1 for x in outs[:rank + 1] if x > 0)
                try:
                    os.rename(tmp, fastk.part_path(dst, part))
                except OSError as x:
                    bad = f"{fastk.part_path(dst, part)}: {x}"
            else:
                os.unlink(tmp)
            gathered = [None] * world if rank == 0 else None
            dist.gather_object((span[0], bcounts, bad), gathered, dst=_global(group, 0), group=group)
            written = 12 + n_out * pbyte if n_out > 0 else 0
            if rank == 0:
                bad = bad or next((g[2] for g in gathered if g[2]), None)
                if bad is None:
                    try:
                        if total == 0:                     # what condition_table writes: the source's part count,
                            nparts = max(src_parts, 1)     # every part empty
                            for q in range(1, nparts + 1):
                                _write_atomic(fastk.part_path(dst, q), struct.pack("<iq", k, 0))
                            written += 12 * nparts
                        index = np.zeros(1 << (8 * ibyte), dtype=np.int64)
                        for s0, c, _ in gathered:
                            index[s0:s0 + len(c)] += c
                        minval = max(minval_src, ethresh) if do_trim else minval_src
                        stub = struct.pack("<4i", k, nparts, minval, ibyte) + np.cumsum(index).astype("<i8").tobytes()
                        _write_atomic(fastk.stub_path(dst), stub)
                        written += len(stub)
                    except OSError as x:
                        bad = f"{fastk.stub_path(dst)}: {x}"
            if max(_reduce([int(bad is not None)], coll, group, dist.ReduceOp.MAX)):
                mine = [part] if part is not None else list(range(1, nparts + 1)) if rank == 0 and total == 0 else []
                for q in mine:
                    if os.path.exists(fastk.part_path(dst, q)):
                        os.unlink(fastk.part_path(dst, q))
                raise _lib.HetmersError(-4, f"rank {rank}: putting {dst} in place failed" + (f": {bad}" if bad else ""))
            if rank == 0:
                for q in range(nparts + 1, old_parts + 1):     # parts an older table of this name had beyond ours
                    if os.path.exists(fastk.part_path(dst, q)):
                        os.unlink(fastk.part_path(dst, q))
            lap("commit", t)
        finally:
            job.close()
            writer.shutdown(wait=True)
            if fd >= 0:
                os.close(fd)
            if os.path.exists(tmp):
                os.unlink(tmp)
        ms["writer_busy"] = busy[0]
        st.update(entries_out=total, rank_entries_out=n_out, part=part, nparts=nparts, bytes_written=written,
                  peak_bytes=torch.cuda.max_memory_allocated(dev) - base, ms=ms)
    return st


def _global(group, r: int) -> int:
    return dist.get_global_rank(group, r) if group is not None else r


def _load_share(kt, lo: int, hi: int, dev):
    """ordinals [lo, hi) of a FastK table (fastk.KtabFiles) unpacked on dev -> (keys, counts, second words or None)"""
    import numpy as np
    from .device import DeviceTable
    if hi > lo:
        d_rec = torch.from_numpy(_share_records(kt, lo, hi)).to(dev)
        d_idx = torch.from_numpy(np.ascontiguousarray(kt.index, dtype=np.int64)).to(dev)
        src = DeviceTable.from_records(kt.kmer, kt.ibyte, d_rec, d_idx, first=lo)
        return src.keys, src.cnt, src.keys_lo
    return (torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int16, device=dev),
            torch.empty(0, dtype=torch.int64, device=dev) if kt.kmer > 32 else None)


def _share_records(kt, lo: int, hi: int):
    """the records of ordinals [lo, hi) of a FastK table (fastk.KtabFiles; the range may span part files)"""
    import numpy as np
    pb = kt.pbyte
    rec = np.empty((hi - lo) * pb, dtype=np.uint8)
    at = start = 0
    for p, pn in enumerate(kt.part_nels):                  # the share's records, part by part
        a, b = max(lo, start), min(hi, start + pn)
        if a < b:
            rec[at:at + (b - a) * pb] = kt.records[p][(a - start) * pb:(b - start) * pb]
            at += (b - a) * pb
        start += pn
    return rec


def _nccl(group) -> bool:
    return dist.get_backend(group) == "nccl"


def _lapper(tm: dict):
    """lap(name, t0): add the ms since t0 to tm[name] -> the time now"""
    def lap(name, t0):
        tm[name] = tm.get(name, 0.0) + (time.perf_counter() - t0) * 1e3
        return time.perf_counter()
    return lap


def _in_place(fn, t: torch.Tensor, group):
    """run collective fn(tensor) on t in place (NCCL), or through a host copy when the backend (gloo) has no
    collective for device tensors"""
    if t.is_cuda and not _nccl(group):
        h = t.cpu()
        fn(h)
        t.copy_(h)
    else:
        fn(t)
    return t


def _all_to_all(out: torch.Tensor, inp: torch.Tensor, out_splits, in_splits, group):
    """all_to_all_single with per-rank splits; device tensors go through host copies on gloo"""
    if out.is_cuda and not _nccl(group):
        h = torch.empty(out.shape, dtype=out.dtype)
        dist.all_to_all_single(h, inp.cpu(), out_splits, in_splits, group=group)
        out.copy_(h)
    else:
        dist.all_to_all_single(out, inp, out_splits, in_splits, group=group)
    return out


def _libc_free(p):
    import ctypes as C
    libc = C.CDLL(None)
    libc.free.argtypes = [C.c_void_p]
    libc.free(p)


def sort_pair_records(recs):
    """sort a structured array of pair records (hetmers.PAIR_DTYPE) in place into the order hm_scan_extract
    returns (hm_sort_pair_records)"""
    from . import _lib
    if len(recs) > 1:
        _lib.lib().hm_sort_pair_records(recs.ctypes.data, len(recs))
    return recs


def gather_pairs(records, dst: int = 0, group=None):
    """the ranks' pair records (structured numpy arrays of hetmers.PAIR_DTYPE, any length, on the host) -> on rank
    `dst` of the group all of them in hm_scan_extract's order (sort_pair_records); None on the other ranks.  Each
    rank's bytes go to dst point-to-point, staged through a device tensor on NCCL."""
    import numpy as np
    from .hetmers import PAIR_DTYPE
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    recs = np.ascontiguousarray(records, dtype=PAIR_DTYPE)
    dev = torch.device("cuda", torch.cuda.current_device()) if _nccl(group) else torch.device("cpu")
    n = torch.tensor([len(recs)], dtype=torch.int64, device=dev)
    every = [torch.empty_like(n) for _ in range(world)]
    dist.all_gather(every, n, group=group)
    sizes = [int(e.item()) for e in every]
    peer = (lambda r: dist.get_global_rank(group, r)) if group is not None else (lambda r: r)   # noqa: E731
    item = PAIR_DTYPE.itemsize
    if rank != dst:
        if sizes[rank] > 0:
            buf = torch.from_numpy(recs.view(np.uint8)).to(dev)
            for w in dist.batch_isend_irecv([dist.P2POp(dist.isend, buf, peer(dst), group)]):
                w.wait()
        return None
    bufs, ops = [], []
    for r in range(world):
        if r == dst or sizes[r] == 0:
            bufs.append(None)
            continue
        bufs.append(torch.empty(sizes[r] * item, dtype=torch.uint8, device=dev))
        ops.append(dist.P2POp(dist.irecv, bufs[-1], peer(r), group))
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()
    parts = [recs if r == dst else bufs[r].cpu().numpy().view(PAIR_DTYPE) for r in range(world) if sizes[r] > 0]
    out = np.concatenate(parts) if parts else np.empty(0, dtype=PAIR_DTYPE)
    return sort_pair_records(np.ascontiguousarray(out))


# ---- extract_kmer_pairs' files written by the ranks (write_pairs, DESIGN.md §6b) ---------------------------------

def read_sma_on_ranks(sma, group, coll):
    """hetmers.read_sma on every rank; a refusal on any rank raises ValueError on every rank -> (pixmap, labels)"""
    from .hetmers import read_sma
    err, res = None, None
    try:
        res = read_sma(sma)
    except ValueError as e:
        err = str(e)
    if dist.get_world_size(group) > 1 and max(_reduce([int(err is not None)], coll, group, dist.ReduceOp.MAX)):
        raise ValueError(err or f"rank {dist.get_rank(group)}: the smudge file {sma} was refused on another rank")
    if err is not None:
        raise ValueError(err)
    return res


def label_paths(out, labels):
    """the output file of every label (a, b): <out>.<a>A<b>B.txt, as extract_kmer_pairs names them"""
    return [f"{out}.{a}A{b}B.txt" for a, b in labels]


def pairs_room(kmer: int, budget: int) -> int:
    """the most records one window may hold under `budget` (hm_pairs_bytes); -1 if not even the fixed part fits"""
    from . import _lib
    f = _lib.lib().hm_pairs_bytes
    if f(kmer, 0) > budget:
        return -1
    lo, hi = 0, max(budget // 24, 1)
    while lo < hi:                                             # the largest r with f(r) <= budget
        mid = (lo + hi + 1) // 2
        if f(kmer, mid) <= budget:
            lo = mid
        else:
            hi = mid - 1
    return lo


def pair_windows(hist, world: int, room: int):
    """The file phase's plan: the fewest passes P such that the key prefixes, cut into P*world windows of near-equal
    record counts (condition_cuts), leave every window within `room` records; window j goes to pass j // world and
    rank j % world.  hist: the records per key prefix, summed over the ranks.  -> (P, cuts [0, ..., len(hist)] of
    P*world + 1 bounds).  A prefix alone above the room is HM_ENOMEM, with the sizes."""
    import numpy as np
    from . import _lib
    h = np.asarray(hist, dtype=np.int64)
    big = int(h.max()) if h.size else 0
    if big > room:
        p = int(np.argmax(h))
        raise _lib.HetmersError(-3, f"writing the pair files: key prefix {p} holds {big} records, beyond the {room} "
                                    f"records one window has room for under the smallest budget of the ranks")
    before = np.concatenate([[0], np.cumsum(h)])
    total = int(before[-1])
    P = max(1, -(-total // (max(room, 1) * world)))
    while True:                                                # ends: with a window per record every window fits
        cuts = condition_cuts(h, P * world)
        if int(np.max(np.diff(before[cuts]))) <= room:
            return P, cuts
        P += 1


def window_segments(counts, rank: int, before, line: int):
    """This rank's segments of one pass: counts[d][s] = lines of label s in the pass's window of rank d (all ranks;
    s = 0 unused), before[s] = lines of label s in every earlier pass.  The window's text holds its labels' lines
    in label order.  -> [(s, offset in the text, bytes, offset in the file of label s)] for its non-empty labels"""
    import numpy as np
    c = np.asarray(counts, dtype=np.int64)
    own = c[rank]
    at = np.concatenate([[0], np.cumsum(own)])
    prior = np.asarray(before, dtype=np.int64) + c[:rank].sum(axis=0)
    return [(s, int(at[s]) * line, int(own[s]) * line, int(prior[s]) * line) for s in range(1, len(own)) if own[s]]


class PairFiles:
    """The label files of one write_pairs call, shared by the ranks: rank 0 creates (truncates) every file, then
    every rank opens them and pwrites its segments at their offsets.  A failure is kept until the next check(), a
    collective: then every rank raises, and rank 0 removes the label files."""

    def __init__(self, paths, group, coll):
        self.paths, self.group, self.coll = list(paths), group, coll
        self.rank = dist.get_rank(group)
        self.fds, self.err = [], None
        if self.rank == 0:
            for p in self.paths:
                try:
                    os.close(os.open(p, os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o666))
                except OSError as x:
                    self.err = f"{p}: {x}"
                    break
        self.check("creating the pair files")                 # (also the barrier after the creation)
        for p in self.paths:
            try:
                self.fds.append(os.open(p, os.O_WRONLY))
            except OSError as x:
                self.err = f"{p}: {x}"
                break
        self.check("opening the pair files")

    def write(self, s: int, data, offset: int):
        """label s's (1-based) bytes at `offset` of its file"""
        if self.err is not None:
            return
        mv = memoryview(data)
        try:
            while len(mv):
                n = os.pwrite(self.fds[s - 1], mv, offset)
                mv, offset = mv[n:], offset + n
        except OSError as x:
            self.err = f"{self.paths[s - 1]}: {x}"

    def check(self, what: str):
        """collective: a failure on any rank so far raises on every rank, rank 0 removing the label files"""
        bad = _reduce([int(self.err is not None)], self.coll, self.group, dist.ReduceOp.MAX)[0] \
            if dist.get_world_size(self.group) > 1 else int(self.err is not None)
        if bad:
            self.fail()
            raise OSError(f"rank {self.rank}: {what} failed on some rank" + (f": {self.err}" if self.err else ""))

    def close(self):
        for fd in self.fds:
            try:
                os.close(fd)
            except OSError as x:
                self.err = self.err or f"close: {x}"
        self.fds = []

    def fail(self):
        """close, and on rank 0 remove every label file (no partial output is left looking complete)"""
        self.close()
        if self.rank == 0:
            for p in self.paths:
                if os.path.exists(p):
                    os.unlink(p)


def write_pair_files(recs, kmer: int, labels, out, group, dev, budget=None, lap=None):
    """The file phase of write_pairs: this rank's pair records (host, any order) -> every rank writes its part of
    `<out>.<a>A<b>B.txt` for every label (a, b) (label s = labels[s - 1]), the files being what extract_kmer_pairs
    writes.  Every rank calls this (DESIGN.md §6b):
      histogram   records per key prefix (hm_k_pairs_hist over the staged records), summed over the ranks
      plan        pair_windows under the smallest room of the ranks (pairs_room of each rank's budget; default: free
                  device memory minus _lib.BUDGET_RESERVE); a prefix above it is HM_ENOMEM on every rank before any
                  file is touched
      per pass    the records staged through the device in chunks of half this rank's room, each chunk's records of
                  the pass routed (hm_k_pairs_route_count / _scatter) and all-to-all'ed to their window's owner, which
                  sorts them (hm_k_pairs_sort), counts lines per label, all-gathers the counts, formats the text
                  (hm_k_pairs_format) and pwrites its segments (window_segments, PairFiles)
    A failure to write on any rank raises on every rank, and rank 0 removes the label files.  -> stats: records (of
    the job), passes, windows, room, chunk, lines per label name, peak device bytes of the phase (torch's allocator;
    its peak statistics are reset), budget"""
    import ctypes as C
    import numpy as np
    from . import _lib
    from .device import _ptr, _stream
    from .hetmers import PAIR_DTYPE
    Lb = _lib.lib()
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    coll = dev if _nccl(group) else torch.device("cpu")
    lap = lap or _lapper({})
    recs = np.ascontiguousarray(recs, dtype=PAIR_DTYPE)
    raw = recs.view(np.uint8)
    item, line, nl = PAIR_DTYPE.itemsize, kmer + 5, len(labels)
    hb = min(_lib.COND_HIST_BITS, 2 * kmer)

    def done(phase, t0):                                       # the phase's kernels have finished
        torch.cuda.synchronize(dev)
        return lap(phase, t0)

    with torch.cuda.device(dev):
        if budget is None:
            budget = torch.cuda.mem_get_info(dev)[0] - _lib.BUDGET_RESERVE
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        t = time.perf_counter()
        own_room = pairs_room(kmer, budget)
        chunk = max(own_room // 2, 1)
        n = len(recs)
        hist = torch.zeros(1 << hb, dtype=torch.int64, device=dev)
        if own_room >= 0:
            for a in range(0, n, chunk):
                d_in = torch.from_numpy(raw[a * item:min(a + chunk, n) * item]).to(dev)
                _lib.check(Lb.hm_k_pairs_hist(_ptr(d_in), d_in.numel() // item, kmer, _ptr(hist), _stream()))
                del d_in
        _in_place(lambda x: dist.all_reduce(x, group=group), hist, group)
        h = hist.cpu().numpy()
        del hist
        room, most = _reduce([own_room, -(-n // chunk)], coll, group, dist.ReduceOp.MIN)[0], \
            _reduce([-(-n // chunk)], coll, group, dist.ReduceOp.MAX)[0]
        if room < 0:
            raise _lib.HetmersError(-3, f"rank {rank}: writing the pair files needs {Lb.hm_pairs_bytes(kmer, 0)} "
                                        f"device bytes per rank before any record; the smallest budget of the ranks "
                                        f"is below that (here {budget})")
        P, cuts = pair_windows(h, world, room)
        wsize = np.diff(np.concatenate([[0], np.cumsum(h)])[cuts])
        t = done("hist_and_plan", t)

        files = PairFiles(label_paths(out, labels), group, coll)
        before = np.zeros(nl + 1, dtype=np.int64)
        cursor_h = np.zeros(world, dtype=np.int64)
        try:
            for p in range(P):
                dest = np.full(1 << hb, -1, dtype=np.int16)
                for d in range(world):
                    dest[cuts[p * world + d]:cuts[p * world + d + 1]] = d
                d_dest = torch.from_numpy(dest).to(dev)
                e = int(wsize[p * world + rank])
                recv = torch.empty(max(e, 1) * item, dtype=torch.uint8, device=dev)
                flag = torch.zeros(1, dtype=torch.int64, device=dev)
                at = 0
                for c in range(most):
                    a, b = min(c * chunk, n), min((c + 1) * chunk, n)
                    d_in = torch.from_numpy(raw[a * item:b * item]).to(dev)
                    counts = torch.zeros(world, dtype=torch.int64, device=dev)
                    _lib.check(Lb.hm_k_pairs_route_count(_ptr(d_in), b - a, kmer, _ptr(d_dest), world, _ptr(counts),
                                                         _stream()))
                    out_c = counts.tolist()
                    cursor_h[1:] = np.cumsum(out_c)[:-1]
                    counts.copy_(torch.from_numpy(cursor_h))
                    ns = sum(out_c)
                    send = torch.empty(max(ns, 1) * item, dtype=torch.uint8, device=dev)
                    _lib.check(Lb.hm_k_pairs_route_scatter(_ptr(d_in), b - a, kmer, _ptr(d_dest), world, _ptr(counts),
                                                           _ptr(send), ns, _ptr(flag), _stream()))
                    del d_in
                    t = done("route", t)
                    sc = torch.tensor(out_c, dtype=torch.int64, device=coll)
                    rc = torch.empty_like(sc)
                    dist.all_to_all_single(rc, sc, group=group)
                    in_c = rc.tolist()
                    nr = sum(in_c)
                    over = at + nr > e                             # (cannot happen: the histogram counted them)
                    tgt = torch.empty(nr * item, dtype=torch.uint8, device=dev) if over else \
                        recv[at * item:(at + nr) * item]
                    _all_to_all(tgt, send[:ns * item], [x * item for x in in_c], [x * item for x in out_c], group)
                    if over:
                        flag.fill_(1)
                    else:
                        at += nr
                    del tgt
                    del send
                    t = done("all_to_all", t)
                if _reduce([int(at != e or flag.item() != 0)], coll, group, dist.ReduceOp.MAX)[0]:
                    raise _lib.HetmersError(-2, f"rank {rank}: pass {p} routed {at} records into a window of {e}")
                del d_dest, flag

                alt = torch.empty_like(recv)
                scratch = torch.empty(max(Lb.hm_pairs_sort_scratch_bytes(e), 1), dtype=torch.uint8, device=dev)
                in_alt = C.c_int()
                _lib.check(Lb.hm_k_pairs_sort(_ptr(recv), _ptr(alt), e, _ptr(scratch), scratch.numel(),
                                              C.byref(in_alt), _stream()))
                srt = alt if in_alt.value else recv
                del scratch, alt, recv
                bounds = torch.zeros(2 * (nl + 1), dtype=torch.int64, device=dev)
                _lib.check(Lb.hm_k_pairs_label_bounds(_ptr(srt), e, nl, _ptr(bounds), _stream()))
                own = (bounds[1::2] - bounds[0::2]).to(coll)
                del bounds
                t = done("sort", t)
                every = torch.zeros((world, nl + 1), dtype=torch.int64, device=coll)
                every[rank] = own
                dist.all_reduce(every, group=group)
                cnt = every.cpu().numpy()
                short = cnt.sum(axis=1) != wsize[p * world:(p + 1) * world]
                if short.any():                                    # (the same verdict on every rank)
                    raise _lib.HetmersError(-2, f"rank {rank}: records of pass {p} on ranks "
                                                f"{np.flatnonzero(short).tolist()} carry no label of the smudge file")
                text = torch.empty(max(e * line, 1), dtype=torch.uint8, device=dev)
                _lib.check(Lb.hm_k_pairs_format(_ptr(srt), e, kmer, _ptr(text), _stream()))
                del srt
                t = done("format", t)
                host = text[:e * line].cpu().numpy()
                del text
                t = lap("text_d2h", t)
                for s, a, nb, off in window_segments(cnt, rank, before, line):
                    files.write(s, host[a:a + nb], off)
                before += cnt.sum(axis=0)
                del host
                t = lap("write", t)
            files.close()
            files.check("writing the pair files")
        except BaseException:
            files.fail()
            raise
        lines = {f"{a}A{b}B": int(before[s + 1]) for s, (a, b) in enumerate(labels)}
        return {"records": int(h.sum()), "passes": P, "windows": P * world, "room": room, "chunk": chunk,
                "chunks": most,
                "lines": lines, "budget": budget, "peak_bytes": torch.cuda.max_memory_allocated(dev) - base}


class StreamedShardedScan:
    """The streamed counterpart of ShardedScan: rank r of the group streams its run-aligned share of the FastK
    table at the path `table` (or the `_lib.HostTable` `table`, whose buffers must outlive the scan, or the
    in-memory fastk.KtabFiles `table`) through `device` under the device budget (`budget` bytes, else free memory
    minus a reserve); no rank holds the table.  from_ktab(L=...) conditions a raw table on the way in.  Pass 2
    settles a Bloom hit on a key another rank owns by asking that rank: the keys go to their owners with
    all_to_all_single, one byte per key comes back (hm_rank_scan_*, DESIGN.md §4c).
    scan() -> the plot (int64[SMAX+1, FMAX+1] on every rank), equal to the in-core scan's; extract(pixmap, dst) ->
    extract_kmer_pairs' records on rank dst, equal to the in-core list.
    list_host_budget (bytes, per rank; None or 0, the default: off) lets a rank whose candidate records and S list
    outgrow its device budget keep them in host memory instead of refusing (DESIGN.md §4c, *Lists in host
    memory*): if any rank's lists go there, every rank's do, and pass 2 runs parked routed rounds, each rank
    answering the queries on the keys it owns against its S list uploaded a partition at a time.  Give it on
    every rank or on none; each rank's lists must stay within its own value (else HetmersError -3 on every rank,
    naming both sizes).  stats["spill"]: this rank's hm_spill_stats (as hetmers.Scan.spill_stats())."""

    def __init__(self, table, group=None, device=None, budget: int | None = None,
                 list_host_budget: int | None = None, _share=None):
        import ctypes as C
        from . import _lib, fastk
        from .hetmers import _host_table
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        dev = torch.device(device if device is not None else "cuda")
        self.device = dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())
        self._coll_dev = self.device if _nccl(group) else torch.device("cpu")
        self.L = L = _lib.lib()
        if isinstance(table, _lib.HostTable):
            self._ht, self._keep = table, None
        elif isinstance(table, fastk.KtabFiles):
            self._ht, self._keep = _host_table(table)
        else:
            self._ht, self._keep = _host_table(fastk.read_ktab(table, mmap=True))   # read again by every scan
        self.kmer = self._ht.kmer
        seeds = common_seeds(self._coll_dev, group)
        sd = (C.c_uint64 * 2)(*seeds)
        if budget is not None:
            L.hm_set_device_budget(int(budget))
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            if _share is None:
                _lib.check(L.hm_rank_scan_create(C.byref(self._ht), self.device.index, self.rank, self.world, sd,
                                                 C.byref(h)))
            else:                                               # table: this rank's share of _share's cuts
                n_total, cuts, first = _share
                _lib.check(L.hm_rank_scan_create_share(C.byref(self._ht), n_total,
                                                       (C.c_int64 * (self.world + 1))(*cuts),
                                                       (C.c_uint64 * self.world)(*first), self.device.index,
                                                       self.rank, self.world, sd, C.byref(h)))
        self._h = h
        self._host_lists = bool(list_host_budget) and int(list_host_budget) > 0
        if self._host_lists:
            _lib.check(L.hm_rank_scan_set_list_host_budget(h, int(list_host_budget)))
        cuts = (C.c_int64 * (self.world + 1))()
        _lib.check(L.hm_rank_scan_cuts(h, cuts, None))
        self.cuts = [int(c) for c in cuts]
        mine = torch.tensor(self.cuts + [int(self._host_lists)], dtype=torch.int64, device=self._coll_dev)
        every = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(every, mine, group=group)
        if any(not torch.equal(e[:-1], mine[:-1]) for e in every):
            self.close()
            raise RuntimeError(f"rank {self.rank}: the ranks computed different shard cuts from the table files "
                               f"({[e[:-1].tolist() for e in every]})")
        if any(int(e[-1]) != self._host_lists for e in every):
            self.close()
            raise ValueError(f"rank {self.rank}: list_host_budget must be given on every rank or on none (given on "
                             f"ranks {[d for d, e in enumerate(every) if int(e[-1])]})")
        self._lists_host = False                                # (list_host_budget) the job's lists in host memory
        self.share = None                                       # (from_ktab) this rank's conditioned share
        self.status = 0
        self._base_stats = {}                                   # what every stats dict starts with (from_ktab)
        self.stats = {}
        self._pass1_done = False                                # candidates, S list and Bloom filter resident

    @classmethod
    def from_ktab(cls, src, group=None, device=None, L=None, budget=None, host_budget=None, list_host_budget=None):
        """The streamed scan of the FastK table `src` as hetmers -e<L> scans it; every rank calls this.  With L the
        table is trimmed and / or symmetrised on the way in, as hm_scan_examine(L) decides on the whole table
        (job_examine), without writing a conditioned copy: each rank conditions one range of key prefixes, cut on
        run boundaries (run_condition_cuts), in the passes of condition_ktab that its device budget allows beside
        its share of the source; it keeps the packed records of its range in host memory as a one-part table
        (self.share: its stub index counts only them) and streams that share on every scan.  A table that needs
        neither step, and L None, give StreamedShardedScan(src): the source files are streamed, no host copy held.
        budget: device bytes per rank, for the conditioning and the scan (default: free memory minus
        _lib.BUDGET_RESERVE); host_budget: host bytes per rank (default: no cap); list_host_budget: as the
        constructor's (host bytes of this rank's lists in the scans, independent of host_budget).  HM_ENOMEM on every rank, with the
        sizes and before the first pass, when a rank's share of the source and one pass do not fit its budget, when
        a rank's conditioned share (records and stub index) exceeds its host_budget, or when a rank cannot allocate
        it.  stats["condition"]: condition_ktab's stats (verdicts, steps, entries in / out, passes, prefix cuts and
        sub-ranges, entries sent / received per pass, peak device bytes, ms per phase), the entry cuts of the
        shares, and host_bytes, what this rank holds once its share is settled (the host budget is checked
        against the histograms' count, which may exceed it by the keys that equal their reverse complement or
        were held on both strands)."""
        import numpy as np
        from . import _lib, fastk
        if L is None:
            out = cls(src, group, device, budget, list_host_budget)
            out._base_stats = {"condition": {"steps": [], "host_bytes": 0}}
            out.stats = dict(out._base_stats)
            return out
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        dev = torch.device(device if device is not None else "cuda")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        coll = dev if _nccl(group) else torch.device("cpu")
        src, ms = str(src), {}
        lap = _lapper(ms)
        with torch.cuda.device(dev):
            cond_budget = budget if budget is not None else torch.cuda.mem_get_info(dev)[0] - _lib.BUDGET_RESERVE
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            kt = fastk.read_ktab(src, mmap=True)
            k, n, ibyte, minval = kt.kmer, kt.nels, kt.ibyte, kt.minval
            job = _RankConditioning(kt, int(L), group, dev, coll, cond_budget, ms)
            del kt
            st = job.st
            if not job.needed():
                job.close()
                torch.cuda.empty_cache()                        # the scan allocates outside torch's cache
                st.update(entries_out=n, host_bytes=0, peak_bytes=torch.cuda.max_memory_allocated(dev) - base, ms=ms)
                out = cls(src, group, device, budget, list_host_budget)
                out._base_stats = {"condition": st}
                out.stats = dict(out._base_stats)
                return out
            job.plan(lambda h, w, hb: run_condition_cuts(h, w, hb, ibyte, k), f"{src} into host shares")

            # the host share, sized by the histograms before the first pass (a bound: settling merges a reverse
            # complement with an equal original, a palindrome with itself)
            t = time.perf_counter()
            pbyte = ((k + 3) >> 2) - ibyte + 2
            ixlen = 1 << (8 * ibyte)
            needs = [job.rank_entries(d) * pbyte + 8 * ixlen for d in range(world)]
            caps = _reduce([(-1 if host_budget is None else int(host_budget)) if d == rank else 0
                            for d in range(world)], coll, group)
            over = [d for d in range(world) if 0 <= caps[d] < needs[d]]
            buf = index = None
            if not over:
                try:
                    buf = np.empty(needs[rank] - 8 * ixlen, dtype=np.uint8)
                    index = np.zeros(ixlen, dtype=np.int64)
                except MemoryError:
                    buf = index = None
            failed = [d for d, f in enumerate(_reduce([int(d == rank and not over and buf is None)
                                                       for d in range(world)], coll, group)) if f]
            if over or failed:
                job.close()
                if over:
                    raise _lib.HetmersError(-3, f"rank {rank}: conditioning {src} into host shares across {world} "
                                                f"ranks holds {needs} host bytes per rank, beyond the host budgets "
                                                f"{caps} of ranks {over} (-1: no cap)")
                raise _lib.HetmersError(-3, f"rank {rank}: conditioning {src} into host shares across {world} "
                                            f"ranks: ranks {failed} cannot allocate their "
                                            f"{[needs[d] for d in failed]} host bytes")
            t = lap("host_alloc", t)
            at, first = 0, None

            def take(rec, keys):
                nonlocal at, first
                if first is None:
                    first = int(keys[0]) & _U64
                torch.from_numpy(buf[at:at + rec.numel()]).copy_(rec)
                at += rec.numel()

            try:
                job.run(take)
            finally:
                job.close()
            torch.cuda.empty_cache()
            t = time.perf_counter()
            m_out = at // pbyte
            buf.resize(at, refcheck=False)         # the histograms count a merged pair of equal keys twice
            s0, s1 = job.span
            index[s0:s1] = job.bcounts
            np.cumsum(index, out=index)

            # every rank's entry cut and first key: an empty rank's first key is the next non-empty rank's, so that
            # it owns no key (~0 past the last)
            got = _reduce(sum(([m_out, _signed(first) if first is not None else 0] if d == rank else [0, 0]
                               for d in range(world)), []), coll, group)
            outs, firsts = got[0::2], [x & _U64 for x in got[1::2]]
            cuts = [0] + np.cumsum(outs).tolist()
            first_keys = [next((firsts[q] for q in range(r, world) if outs[q] > 0), _U64) for r in range(world)]
            lap("host_share", t)
            st.update(entries_out=cuts[-1], rank_entries_out=m_out, cuts=cuts, host_bytes=buf.nbytes + index.nbytes,
                      peak_bytes=torch.cuda.max_memory_allocated(dev) - base, ms=ms)
            share = fastk.KtabFiles(kmer=k, nparts=1, minval=max(minval, int(L)) if job.do_trim else minval,
                                    ibyte=ibyte, index=index, part_nels=[m_out], records=[buf])
        out = cls(share, group, device, budget, list_host_budget, _share=(cuts[-1], cuts, first_keys))
        out.share = share
        out._base_stats = {"condition": st}
        out.stats = dict(out._base_stats)
        return out

    def _view(self, ptr: int, nbytes: int) -> torch.Tensor:
        return _cuda_view(ptr, max(nbytes, 1), self.device)[:nbytes]

    def _lap(self, tm):
        return _lapper(tm)

    def _sync(self):
        torch.cuda.synchronize(self.device)                    # (the library works on its own streams)

    def _pass1(self, lap):
        """pass 1 over this rank's share, the job-wide fingerprint verdict (HM_EUNSUPPORTED on every rank for an
        asymmetric table), the S index and the Bloom segments all-gathered in place -> (candidates, max_slice)"""
        import ctypes as C
        from . import _lib
        L, h, g, W = self.L, self._h, self.group, self.world
        if self._host_lists:
            return self._pass1_host(lap)
        self._pass1_done = False
        t = time.perf_counter()
        fp = (C.c_uint64 * 4)()
        _lib.check(L.hm_rank_scan_pass1(h, fp))
        t = lap("pass1", t)
        acc = torch.tensor([v - (1 << 64) if v >= (1 << 63) else v for v in fp], dtype=torch.int64,
                           device=self._coll_dev)
        symmetric = fingerprint_verdict(acc, g)
        nc, ms = C.c_int64(), C.c_int64()
        _lib.check(L.hm_rank_scan_prepare(h, int(symmetric), C.byref(nc), C.byref(ms)))
        t = lap("verdict_and_s_index", t)
        seg, segb = C.c_void_p(), C.c_int64()
        _lib.check(L.hm_rank_scan_bloom(h, C.byref(seg), C.byref(segb)))
        if W > 1:
            view = self._view(seg.value, W * segb.value).view(W, segb.value)
            _in_place(lambda x: exchange_segments(x, self.rank, g), view, g)
            self._sync()
        lap("bloom_allgather", t)
        self._pass1_done = True
        return nc.value, ms.value

    def _pass1_host(self, lap):
        """_pass1 of ranks with a list host budget: one mode for the job -- if any rank's lists went to host memory
        in pass 1, every rank's go there (hm_rank_scan_host_lists) and prepare builds no S index -- with a failure
        on any rank (its lists over its list_host_budget, a plan refusal) raised on every rank"""
        import ctypes as C
        from . import _lib
        L, h, g, W = self.L, self._h, self.group, self.world
        self._pass1_done = self._lists_host = False
        t = time.perf_counter()
        fp = (C.c_uint64 * 4)()
        err = None
        try:
            _lib.check(L.hm_rank_scan_pass1(h, fp))
        except _lib.HetmersError as e:
            err = e
        spilled = err is None and self.spill_stats()["spilled"]
        t = lap("pass1", t)
        symmetric, self._lists_host = pass1_agreement(list(fp), spilled, None if err is None else err,
                                                      self._coll_dev, g)
        nc, ms = C.c_int64(), C.c_int64()
        err = None
        try:
            if self._lists_host:
                _lib.check(L.hm_rank_scan_host_lists(h))
            _lib.check(L.hm_rank_scan_prepare(h, int(symmetric), C.byref(nc), C.byref(ms)))
        except _lib.HetmersError as e:
            err = e
        raise_on_any_rank(err, "preparing pass 2", self._coll_dev, g)
        t = lap("verdict_and_s_index", t)
        seg, segb = C.c_void_p(), C.c_int64()
        _lib.check(L.hm_rank_scan_bloom(h, C.byref(seg), C.byref(segb)))
        if W > 1:
            view = self._view(seg.value, W * segb.value).view(W, segb.value)
            _in_place(lambda x: exchange_segments(x, self.rank, g), view, g)
            self._sync()
        lap("bloom_allgather", t)
        self._pass1_done = True
        return nc.value, ms.value

    def spill_stats(self) -> dict:
        """this rank's hm_spill_stats (hm_rank_scan_spill_stats), as hetmers.Scan.spill_stats() gives them"""
        import ctypes as C
        from . import _lib
        st = _lib.SpillStats()
        _lib.check(self.L.hm_rank_scan_spill_stats(self._h, C.byref(st)))
        return st.as_dict()

    def _rounds(self, n_cand, max_slice, slices_fn, route_fn, settle_fn, lap):
        """the slice every rank can hold, its buffers (slices_fn), then every round up to the most any rank needs:
        route_fn(round, counts) -> the query keys all-to-all'ed to their owners -> answer -> the answer bytes
        all-to-all'ed back -> settle_fn().  -> (rounds, slice, queries sent to each rank)"""
        import ctypes as C
        from . import _lib
        L, h, g, W = self.L, self._h, self.group, self.world
        kw = 2 if self.kmer > 32 else 1
        t = time.perf_counter()
        lim = torch.tensor([max_slice, -n_cand], dtype=torch.int64, device=self._coll_dev)
        dist.all_reduce(lim, op=dist.ReduceOp.MIN, group=g)
        slice_ = max(1, min(int(lim[0]), -int(lim[1])))        # the smallest room, no more than the most candidates
        rounds = C.c_int64()
        ptr = [C.c_void_p() for _ in range(4)]
        if self._host_lists:
            err = None
            try:
                _lib.check(slices_fn(h, slice_, C.byref(rounds), *[C.byref(p) for p in ptr]))
            except _lib.HetmersError as e:
                err = e
            raise_on_any_rank(err, "sizing pass 2's buffers", self._coll_dev, g)
        else:
            _lib.check(slices_fn(h, slice_, C.byref(rounds), *[C.byref(p) for p in ptr]))
        rt = torch.tensor([rounds.value], dtype=torch.int64, device=self._coll_dev)
        dist.all_reduce(rt, op=dist.ReduceOp.MAX, group=g)
        n_rounds = int(rt.item())
        q = 2 * slice_
        # lists in host memory: every rank's queries go to their owners, this rank's own included
        senders = W if self._lists_host else W - 1
        send = self._view(ptr[0].value, 8 * kw * q).view(torch.int64)
        recv = self._view(ptr[1].value, 8 * kw * q * senders).view(torch.int64)
        ans_recv = self._view(ptr[2].value, q * senders)
        ans_sent = self._view(ptr[3].value, q)
        t = lap("slices", t)
        counts = (C.c_int64 * W)()
        sent_to = [0] * W
        for rd in range(n_rounds):
            _lib.check(route_fn(h, rd, counts))
            t = lap("resolve", t)
            if W == 1 and self._lists_host:                     # the one rank answers itself
                ns = nr = int(counts[0])
                sent_to[0] += ns
                recv[:kw * nr].copy_(send[:kw * ns])
                self._sync()
                t = lap("exchange_queries", t)
                _lib.check(L.hm_rank_scan_answer(h, nr))
                t = lap("answer", t)
                ans_sent[:ns].copy_(ans_recv[:nr])
                self._sync()
                t = lap("exchange_answers", t)
            elif W > 1:
                out_c = [int(c) for c in counts]
                sc = torch.tensor(out_c, dtype=torch.int64, device=self._coll_dev)
                rc = torch.empty_like(sc)
                dist.all_to_all_single(rc, sc, group=g)
                in_c = [int(c) for c in rc.tolist()]
                ns, nr = sum(out_c), sum(in_c)
                for r_, c in enumerate(out_c):
                    sent_to[r_] += c
                _all_to_all(recv[:kw * nr], send[:kw * ns], [kw * c for c in in_c], [kw * c for c in out_c], g)
                self._sync()
                t = lap("exchange_queries", t)
                _lib.check(L.hm_rank_scan_answer(h, nr))
                t = lap("answer", t)
                _all_to_all(ans_sent[:ns], ans_recv[:nr], out_c, in_c, g)
                self._sync()
                t = lap("exchange_answers", t)
            _lib.check(settle_fn(h))
            t = lap("settle", t)
        return n_rounds, slice_, sent_to

    def scan(self, timings: dict | None = None) -> torch.Tensor:
        import ctypes as C
        from . import _lib
        L, h, g, W = self.L, self._h, self.group, self.world
        lap = self._lap({} if timings is None else timings)
        with torch.cuda.device(self.device):
            nc, ms = self._pass1(lap)
            n_rounds, slice_, sent_to = self._rounds(nc, ms, L.hm_rank_scan_slices, L.hm_rank_scan_route,
                                                     L.hm_rank_scan_settle, lap)
            t = time.perf_counter()
            dp, st = C.c_void_p(), C.c_uint64()
            _lib.check(L.hm_rank_scan_result(h, C.byref(dp), C.byref(st)))
            plot = self._view(dp.value, 8 * _lib.PLOT_CELLS).view(torch.int64)
            if W > 1:
                _in_place(lambda x: allreduce_plot(x, g), plot, g)
                self._sync()
            out = plot.clone().view(_lib.SMAX + 1, _lib.PLOT_W)
            lap("plot_allreduce", t)
        self.status = int(st.value)
        self.stats = {**self._base_stats, "rounds": n_rounds, "slice": slice_, "max_slice": ms, "candidates": nc,
                      "queries_sent_to": sent_to, "spill": self.spill_stats()}
        if self._host_lists and not self.symm_ok():
            raise _lib.HetmersError(-2, f"rank {self.rank}: the streamed scan ended with a non-zero status word on some "
                                        f"rank (here {self.status:#x}); its plot must not be used")
        return out

    def extract(self, pixmap, dst: int = 0, timings: dict | None = None):
        """extract_kmer_pairs' pair list for a pixel -> smudge map (uint16[SMAX+1, FMAX+1], label 0 = none): on rank
        `dst` the structured array hetmers.Scan.extract returns for the table, the same records in the same order;
        None on the other ranks.  Reuses the candidates of the last scan() (or extract()) when every rank left a
        clean pass 1, else runs pass 1 first.  A Bloom hit on a key another rank owns is settled by that rank, as
        in scan(); the records each rank lists are gathered on dst (gather_pairs).  stats["pass1_reused"] tells
        which happened."""
        lap = self._lap({} if timings is None else timings)
        recs = self._list_pairs(pixmap, lap, True)
        t = time.perf_counter()
        res = gather_pairs(recs, dst, self.group)
        lap("gather_and_sort", t)
        return res

    def write_pairs(self, sma, out, timings: dict | None = None, budget: int | None = None):
        """extract_kmer_pairs' output files for the smudges of `sma`, as ShardedScan.write_pairs writes them; every
        rank calls this.  The pairs are listed as extract() lists them (the same pass-1 reuse and refusals), but each
        rank's records are handed over unsorted (hm_rank_scan_extract_records) to the file phase (write_pair_files),
        which sorts them on the GPUs.  budget: device bytes per rank for the file phase (default: free device memory
        minus _lib.BUDGET_RESERVE, beside what the streamed scan holds).  -> the file phase's stats, on every rank;
        timings (ms): the listing's phases, then hist_and_plan, route, all_to_all, sort, format, text_d2h, write"""
        pix, labels = read_sma_on_ranks(sma, self.group, self._coll_dev)
        lap = self._lap({} if timings is None else timings)
        recs = self._list_pairs(pix, lap, False)
        with torch.cuda.device(self.device):
            return write_pair_files(recs, self.kmer, labels, out, self.group, self.device, budget, lap)

    def _list_pairs(self, pixmap, lap, sort: bool):
        """the routed listing of extract(): this rank's records (host; sorted as hm_scan_extract sorts them, or in the
        order listed) and self.stats; raises on every rank when a status word is dirty on any"""
        import ctypes as C
        import numpy as np
        from . import _lib
        from .hetmers import PAIR_DTYPE
        L, h, g = self.L, self._h, self.group
        pm = np.ascontiguousarray(pixmap, dtype=np.uint16).reshape(-1)
        if pm.size != _lib.PLOT_CELLS:
            raise ValueError(f"pixmap has {pm.size} cells, not {_lib.PLOT_CELLS}")
        with torch.cuda.device(self.device):
            reuse = self._pass1_done and self.status == 0
            if self.world > 1:                                  # (every rank must take the same branch)
                bad = torch.tensor([int(not reuse)], dtype=torch.int32, device=self._coll_dev)
                dist.all_reduce(bad, op=dist.ReduceOp.MAX, group=g)
                reuse = int(bad.item()) == 0
            if not reuse:
                self.status = 0
                self._pass1(lap)
            t = time.perf_counter()
            nc, ms = C.c_int64(), C.c_int64()
            if self._host_lists:
                err = None
                try:
                    _lib.check(L.hm_rank_scan_extract_prepare(h, pm.ctypes.data, C.byref(nc), C.byref(ms)))
                except _lib.HetmersError as e:
                    err = e
                raise_on_any_rank(err, "preparing the pair listing", self._coll_dev, g)
            else:
                _lib.check(L.hm_rank_scan_extract_prepare(h, pm.ctypes.data, C.byref(nc), C.byref(ms)))
            lap("extract_prepare", t)
            n_rounds, slice_, sent_to = self._rounds(nc.value, ms.value, L.hm_rank_scan_extract_slices,
                                                     L.hm_rank_scan_extract_route, L.hm_rank_scan_extract_settle, lap)
            t = time.perf_counter()
            out, n, st = C.POINTER(_lib.PairRec)(), C.c_int64(), C.c_uint64()
            take = L.hm_rank_scan_extract_result if sort else L.hm_rank_scan_extract_records
            _lib.check(take(h, C.byref(out), C.byref(n), C.byref(st)))
            recs = np.empty(n.value, dtype=PAIR_DTYPE)
            if n.value:
                C.memmove(recs.ctypes.data, out, n.value * PAIR_DTYPE.itemsize)
            _libc_free(out)
            lap("rank_sort" if sort else "rank_records", t)
        self.status = int(st.value)
        self.stats = {**self._base_stats, "rounds": n_rounds, "slice": slice_, "max_slice": ms.value,
                      "candidates": nc.value, "queries_sent_to": sent_to, "pass1_reused": reuse,
                      "records": int(n.value), "spill": self.spill_stats()}
        if self._host_lists and not self.symm_ok():
            raise _lib.HetmersError(-2, f"rank {self.rank}: the routed pair listing ended with a non-zero status word on "
                                        f"some rank (here {self.status:#x}); its records must not be used")
        if not self.symm_ok():
            raise RuntimeError(f"rank {self.rank}: the routed pair listing ended with a non-zero status word on some "
                               f"rank (here {self.status:#x}); its records must not be used")
        return recs

    def residency(self):
        """-> (peak device bytes since the last scan began, its chunks, the budget)"""
        import ctypes as C
        b, c, bud = C.c_int64(), C.c_int64(), C.c_int64()
        from . import _lib
        _lib.check(self.L.hm_rank_scan_residency(self._h, C.byref(b), C.byref(c), C.byref(bud)))
        return b.value, c.value, bud.value

    def symm_ok(self) -> bool:
        """status words of the last scan on every rank: all clean?"""
        bad = torch.tensor([int(self.status != 0)], dtype=torch.int32, device=self._coll_dev)
        if self.world > 1:
            dist.all_reduce(bad, op=dist.ReduceOp.MAX, group=self.group)
        return int(bad.item()) == 0

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            with torch.cuda.device(self.device):
                self.L.hm_rank_scan_destroy(self._h)
        self._h = None
        self._keep = self.share = None                         # the host buffers the scan streamed
