"""Multi-GPU plumbing for the check path: one process per GPU (torch.distributed).

The path shards by CHECK: every rank holds a replica of the snapshot (100 M tuples are
~2 GB, far below one GPU's HBM) and answers its own slice of the batch; there is no
data-path collective (SURVEY.md 8e, DESIGN.md 7). The only communication is the
all-gather that returns the answers to the caller's order, plus the max-reduce of the
timings in bench.py. Works with backend "nccl" (GPU tensors) and "gloo" (CPU tensors;
used by the world_size-2 tests, where the evaluator is a stub).
"""
from __future__ import annotations

from typing import Callable

import numpy as np
import torch
import torch.distributed as dist

from ._lib import CHECK_DTYPE


def shard_bounds(n: int, rank: int, world: int):
    """Contiguous, balanced slice of n items for this rank."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class ShardedChecker:
    """check_bulk over a process group: slice, answer locally, all-gather the answers.

    evaluate: callable(items ndarray) -> uint8 ndarray; on GPU ranks this is
    `engine.check_bulk`. Every rank must call check_bulk with the same items.
    """

    def __init__(self, evaluate: Callable[[np.ndarray], np.ndarray], group=None, device: str | None = None):
        self.evaluate = evaluate
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.device = device or ("cuda" if dist.get_backend(group) == "nccl" else "cpu")

    def check_bulk(self, items: np.ndarray) -> np.ndarray:
        n = items.size
        lo, hi = shard_bounds(n, self.rank, self.world)
        mine = self.evaluate(items[lo:hi]) if hi > lo else np.empty(0, dtype=np.uint8)
        width = -(-n // self.world)  # every rank contributes a fixed-width block
        block = torch.zeros(width, dtype=torch.uint8)
        block[: hi - lo] = torch.from_numpy(np.ascontiguousarray(mine))
        block = block.to(self.device)
        gathered = [torch.empty_like(block) for _ in range(self.world)]
        dist.all_gather(gathered, block, group=self.group)
        out = np.empty(n, dtype=np.uint8)
        for r, t in enumerate(gathered):
            rlo, rhi = shard_bounds(n, r, self.world)
            out[rlo:rhi] = t[: rhi - rlo].cpu().numpy()
        return out


def max_over_ranks(value: float, group=None, device: str = "cpu") -> float:
    """Timings are reported as the max over ranks (bench.py contract)."""
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t.item())


# ---------------------------------------------------------------------------------------------
# Object-hash sharded STORE (north-star's other multi-GPU mode; SURVEY.md 8e, DESIGN.md 7), device resident.
#
# Every rank owns the relationships whose resource id % world == rank. A check starts on the owner of its
# resource; an edge to an object of another shard (or into a non-pure permission) is raised as a sub-query. Ranks
# run pass by pass until no rank raises any; values then travel back level by level and are folded into the jobs
# that raised them. Cross-shard traffic is 16 B per sub-query out, 1 B back.
#
# Per level: ONE kernel pass over the level's queries (zg_shard_pass_dev), a counting-sort kernel that bucketises
# the raised sub-queries by owner (zg_shard_route_dev), an N-int count exchange and one all-to-all of the 16-byte
# sub-queries, device buffer to device buffer (NCCL over NVLink). Values (1 byte per sub-query) travel back with
# the reverse all-to-all and are OR-ed into the (query, leaf) that raised them by a kernel that reads them in
# routed order (zg_shard_fold_dev). Nothing is staged through the host; the host sees N counts per level.


class TorchDeviceTransport:
    """Ragged all-to-all of tensors over torch.distributed: CUDA tensors over nccl, or CPU tensors over gloo
    (device=torch.device("cpu"))."""

    def __init__(self, group=None, device=None):
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.device = device or torch.device("cuda", torch.cuda.current_device())

    def exchange_counts(self, counts):
        t = torch.tensor(counts, dtype=torch.int64, device=self.device)
        r = torch.empty_like(t)
        dist.all_to_all_single(r, t, group=self.group)
        return [int(x) for x in r.cpu()]

    def alltoall(self, send: torch.Tensor, send_counts, recv_counts, width: int) -> torch.Tensor:
        """send: uint8 tensor of sum(send_counts) * width bytes, destination-major."""
        out = torch.empty(sum(recv_counts) * width, dtype=torch.uint8, device=self.device)
        dist.all_to_all_single(out, send, output_split_sizes=[c * width for c in recv_counts],
                               input_split_sizes=[c * width for c in send_counts], group=self.group)
        if self.device.type == "cuda":
            torch.cuda.current_stream().synchronize()  # the engine's calls run on its own stream
        return out

    def allreduce_sum(self, x: int) -> int:
        t = torch.tensor([int(x)], dtype=torch.int64, device=self.device)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return int(t.item())


class LocalDeviceTransport:
    """`world` virtual ranks in ONE process on ONE GPU (threads): tensors change hands by reference. Tests the
    device-resident protocol without NCCL. Build with LocalDeviceTransport.cluster(world)."""

    def __init__(self, rank, world, shared, device=None):
        self.rank, self.world, self._s = rank, world, shared
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())

    def _sync(self):
        if self.device.type == "cuda":
            torch.cuda.current_stream().synchronize()

    @staticmethod
    def cluster(world, device=None):
        """device=torch.device("cpu"): host tensors (the kernel emulator of tests/emu drives the same protocol)."""
        import threading

        shared = {"box": [None] * world, "bar": threading.Barrier(world), "sum": [0] * world}
        return [LocalDeviceTransport(r, world, shared, device) for r in range(world)]

    def exchange_counts(self, counts):
        s = self._s
        s["box"][self.rank] = list(counts)
        s["bar"].wait()
        out = [s["box"][src][self.rank] for src in range(self.world)]
        s["bar"].wait()
        return out

    def alltoall(self, send, send_counts, recv_counts, width):
        s = self._s
        offs = np.concatenate([[0], np.cumsum(send_counts)]) * width
        self._sync()
        s["box"][self.rank] = [send[int(offs[d]):int(offs[d + 1])] for d in range(self.world)]
        s["bar"].wait()
        parts = [s["box"][src][self.rank] for src in range(self.world)]
        out = torch.cat(parts) if parts else torch.empty(0, dtype=torch.uint8, device=self.device)
        self._sync()
        s["bar"].wait()
        return out

    def allreduce_sum(self, x):
        s = self._s
        s["sum"][self.rank] = int(x)
        s["bar"].wait()
        tot = sum(s["sum"])
        s["bar"].wait()
        return tot


class DeviceShardedChecker:
    """CheckBulkPermissions over an object-hash sharded store, device resident. Every rank brings ITS OWN batch
    (a CUDA uint8 tensor of n x 16 bytes) and gets the answers of that batch (CUDA uint8 tensor of n codes):
    checks are routed to the owner of their resource, evaluated level by level across the shards, and the
    answers routed back."""

    ITEM = 16

    def __init__(self, engine, transport):
        self.e, self.t = engine, transport
        self.stats = {"levels": 0, "subqueries_sent": 0, "bytes_sent": 0, "exchanges": 0}

    def _route(self, d_items: int, n: int, level: int):
        """-> (routed uint8 tensor, src int32 tensor, send_counts, recv_counts)"""
        dev, w = self.t.device, self.t.world
        routed = torch.empty(max(n, 1) * self.ITEM, dtype=torch.uint8, device=dev)
        src = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        counts = self.e.shard_route_dev(d_items, n, level, w, routed.data_ptr(), src.data_ptr())
        return routed[: n * self.ITEM], src[:n], counts, self.t.exchange_counts(counts)

    def check_bulk(self, d_items: torch.Tensor, n: int, no_wildcards: bool = False) -> torch.Tensor:
        """no_wildcards: every pass of every rank evaluates with the wildcard relationships invisible (LookupSubjects'
        second verification; the sub-queries raised to other shards are evaluated the same way)."""
        dev, t = self.t.device, self.t
        shard_pass = self.e.shard_pass_nowild_dev if no_wildcards else self.e.shard_pass_dev
        # level "-1": this rank's own batch goes to the owners of its resources
        routed, src0, sc, rc = self._route(d_items.data_ptr(), n, -1)
        queries = t.alltoall(routed, sc, rc, self.ITEM)
        self.stats["exchanges"] += 1
        levels = [{"src": src0, "send": sc, "recv": rc}]  # routing that produced level lv's queries
        lv = 0
        while True:
            nq = queries.numel() // self.ITEM
            nsub = shard_pass(queries.data_ptr() if nq else 0, nq, lv)
            routed, src, sc, rc = self._route(0, nsub, lv)
            nxt = t.alltoall(routed, sc, rc, self.ITEM)
            self.stats["exchanges"] += 1
            self.stats["subqueries_sent"] += int(nsub)
            self.stats["bytes_sent"] += int(nsub) * self.ITEM
            levels.append({"src": src, "send": sc, "recv": rc, "nq": nq, "nsub": int(nsub)})
            queries = nxt
            lv += 1
            if t.allreduce_sum(queries.numel()) == 0:
                break
            if lv > 60:
                raise RuntimeError("sharded check did not converge within the dispatch depth")
        self.stats["levels"] = max(self.stats["levels"], lv)
        # values flow back: level lv's outputs answer the sub-queries level lv-1 raised
        out_next = torch.empty(0, dtype=torch.uint8, device=dev)  # outputs of the (empty) deepest level
        for k in range(lv - 1, -1, -1):
            L = levels[k + 1]
            # out_next holds one byte per query that ARRIVED at level k+1, source-major: send them home
            back = t.alltoall(out_next, L["recv"], L["send"], 1)
            self.stats["bytes_sent"] += int(back.numel())
            out = torch.empty(max(L["nq"], 1), dtype=torch.uint8, device=dev)
            self.e.shard_fold_dev(k, back.data_ptr() if L["nsub"] else 0, L["src"].data_ptr() if L["nsub"] else 0, L["nsub"],
                                  out.data_ptr(), final_codes=(k == 0))
            out_next = out[: L["nq"]]
        # level 0's outputs answer the checks that were routed here: back to their callers, in the callers' order
        home = t.alltoall(out_next, levels[0]["recv"], levels[0]["send"], 1)
        answers = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        self.e.shard_unroute_dev(levels[0]["src"].data_ptr() if n else 0, home.data_ptr() if n else 0, n, answers.data_ptr())
        return answers[:n]


# ---------------------------------------------------------------------------------------------
# LookupResources over the object-hash sharded store (DESIGN.md 4 and 7).
#
# Shard k holds the relationships whose resource it owns, so every object it discovers in its own reverse rows is
# an object it owns: each rank dedups what it discovers with its own visited slices, and each object enters the
# frontier once. A level is a local expand of the WHOLE replicated frontier on every rank, then an all-gather of
# the new entries (one count exchange that also carries the overflow flag, one all-to-all). Candidates start on
# their owner, are verified by the sharded check protocol, and the answers go home with one more all-to-all.

MAX_DEPTH = 50  # ZG_MAX_DEPTH (include/zgpu.h): the walk expands levels 0 .. MAX_DEPTH + 1, as a replica's does
LOOKUP_ROUND = 64  # lookups per round (visited slices; the lookup index in an answer key has 6 bits)
WILDCARDS_INCLUDE = 0  # ZG_WILDCARDS_INCLUDE (include/zgpu.h)


class DeviceShardedLookup:
    """LookupResources over an object-hash sharded store, device resident. `lookup_resources` is collective: every
    rank brings its own list of requests (possibly empty) and gets one answer per request of its own."""

    REQ = np.dtype([("subj", "<u4"), ("res_type", "<u2"), ("perm", "<u2"), ("stype", "<u2"), ("srel", "<u2")])

    def __init__(self, engine, transport, walk_cap: int = 1 << 22, checker: DeviceShardedChecker | None = None,
                 verify_chunk: int = 1 << 16):
        """walk_cap: entries of a frontier and of the walk's candidates on one rank; a round that overflows it is
        redone in halves, and a single lookup then verifies every resource of its type the rank owns. verify_chunk:
        candidates per check_bulk call, so that their raised sub-queries fit the engine's sub-query buffer."""
        self.e, self.t, self.walk_cap, self.verify_chunk = engine, transport, int(walk_cap), int(verify_chunk)
        self.checker = checker or DeviceShardedChecker(engine, transport)
        # entries_sent / admitted / nowild_verified: LookupSubjects' walk entries sent to other ranks, objects admitted
        # into a frontier by their owner, and items of the no-wildcards verification
        self.stats = {"rounds": 0, "levels": 0, "frontier_entries": 0, "frontier_bytes": 0, "bytes_sent": 0,
                      "candidates": 0, "fallbacks": 0, "halvings": 0, "entries_sent": 0, "admitted": 0, "nowild_verified": 0}

    def _gather_requests(self, mine):
        """Every rank's requests (structured array `mine` of this rank's) -> (all of them in rank order, on every rank;
        the home rank of each; the index of this rank's first)."""
        t, w = self.t, self.t.world
        counts = t.exchange_counts([mine.size] * w)  # requests of every rank, in rank order
        send = torch.from_numpy(np.tile(mine.view(np.uint8), w)).to(t.device)
        got = t.alltoall(send, [mine.size] * w, counts, mine.dtype.itemsize)
        self.stats["bytes_sent"] += mine.size * mine.dtype.itemsize * (w - 1)
        every = got.cpu().numpy().view(mine.dtype)
        return every, np.repeat(np.arange(w, dtype=np.uint8), counts), sum(counts[: t.rank])

    def _verify(self, items, n, no_wildcards=False):
        """Codes of this rank's n check items, in chunks that bound the check protocol's sub-query buffers; every rank
        runs as many chunks as the rank with the most items (check_bulk is collective)."""
        t, w, dev = self.t, self.t.world, self.t.device
        item = DeviceShardedChecker.ITEM
        codes = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        for lo in range(0, max(t.exchange_counts([n] * w)), self.verify_chunk):
            m = max(0, min(self.verify_chunk, n - lo))
            codes[lo:lo + m] = self.checker.check_bulk(items[lo * item:(lo + m) * item] if m else items, m, no_wildcards)
        # the copies into `codes` run on torch's stream, the engine reads `codes` on its own: they must have landed
        # (and the chunks' answer tensors they read must not be handed out again) before the engine's next call
        if dev.type == "cuda":
            torch.cuda.current_stream().synchronize()
        return codes

    def lookup_resources(self, reqs) -> list:
        """reqs: [(res_type_id, perm_slot, subj_type_id, subj_id, subj_rel_slot)] of this rank (subj_rel_slot = SREL_NONE
        for a plain subject). -> per request an ascending uint32 array of resource ids, or None where
        zg_lookup_resources would return ZG_EDEPTH (a candidate could not be decided)."""
        mine = np.zeros(len(reqs), self.REQ)
        for i, (rt, perm, st, subj, srel) in enumerate(reqs):
            mine[i] = (subj, rt, perm, st, srel)
        every, home, first = self._gather_requests(mine)
        out = [None] * mine.size
        for lo in range(0, every.size, LOOKUP_ROUND):
            self._round(every[lo:lo + LOOKUP_ROUND], home[lo:lo + LOOKUP_ROUND], lo - first, out)
        return out

    def _round(self, reqs, home, base, out):
        """One round of <= 64 lookups on every rank; answers of this rank's lookups go to out[base + k]."""
        t, w, dev = self.t, self.t.world, self.t.device
        K = reqs.size
        self.stats["rounds"] += 1
        protos = np.zeros(K, CHECK_DTYPE)
        protos["subj"], protos["perm"], protos["stype"], protos["srel"] = reqs["subj"], reqs["perm"], reqs["stype"], reqs["srel"]
        front = torch.empty(K * 8, dtype=torch.uint8, device=dev)
        nxt = torch.empty(self.walk_cap * 8, dtype=torch.uint8, device=dev)
        self.e.shard_lookup_begin_dev(reqs["res_type"], protos, home, self.walk_cap, front.data_ptr())
        n_in, level, overflow = K, 0, False
        while True:
            n_out, ovf = self.e.shard_lookup_expand_dev(front.data_ptr(), n_in, level, nxt.data_ptr())
            got = t.exchange_counts([2 * n_out + int(ovf)] * w)  # new entries, overflow flag in bit 0
            self.stats["levels"] += 1
            if any(g & 1 for g in got):
                overflow = True
                break
            rc = [g >> 1 for g in got]
            n_in = sum(rc)
            if n_in == 0 or level == MAX_DEPTH + 1:
                break
            # all-gather: this rank's new entries to every rank (itself included), the gathered frontier back
            front = t.alltoall(nxt[: n_out * 8].repeat(w), [n_out] * w, rc, 8)
            self.stats["frontier_entries"] += n_out
            self.stats["frontier_bytes"] += n_out * 8 * (w - 1)
            level += 1
        if overflow and K > 1:
            self.stats["halvings"] += 1
            h = K // 2
            self._round(reqs[:h], home[:h], base, out)
            self._round(reqs[h:], home[h:], base + h, out)
            return
        if overflow:
            self.stats["fallbacks"] += 1
        need = self.e.shard_lookup_candidates_dev(overflow, 0, 0)
        items = torch.empty(max(need, 1) * DeviceShardedChecker.ITEM, dtype=torch.uint8, device=dev)
        n = self.e.shard_lookup_candidates_dev(overflow, items.data_ptr(), need)
        self.stats["candidates"] += n
        codes = self._verify(items, n)
        routed = torch.empty(max(n, 1) * 8, dtype=torch.uint8, device=dev)
        sc = self.e.shard_lookup_route_dev(codes.data_ptr() if n else 0, n, w, routed.data_ptr())
        rc = t.exchange_counts(sc)
        keys = t.alltoall(routed[: sum(sc) * 8], sc, rc, 8)
        self.stats["bytes_sent"] += (sum(sc) - sc[t.rank]) * 8
        nk = sum(rc)
        ids = torch.empty(max(nk, 1) * 4, dtype=torch.uint8, device=dev)
        per, err = self.e.shard_lookup_finish_dev(keys.data_ptr() if nk else 0, nk, ids.data_ptr(), K)
        host = ids[: sum(per) * 4].cpu().numpy().view(np.uint32)
        off = 0
        for k in range(K):
            if home[k] == t.rank:
                out[base + k] = None if (err >> k) & 1 else host[off:off + per[k]].copy()
            off += per[k]

    # -----------------------------------------------------------------------------------------
    # LookupSubjects (DESIGN.md 4 and 7). Shard k holds the forward rows of the objects it owns, but the subjects in
    # those rows can be owned by any shard: each level, every rank expands its own frontier, sends what it finds to
    # the owners (a count exchange that also carries the overflow flag and whether the rank had a frontier, then one
    # all-to-all of 8-byte entries), and each owner admits an object once per lookup. Each rank's candidates are then
    # its batch of check_bulk; the probe verdicts travel to every rank once per round, the HAS candidates of granted
    # lookups are verified again without wildcards, and the answers go home with one more all-to-all.

    SUBJ_REQ = np.dtype([("res", "<u4"), ("res_type", "<u2"), ("perm", "<u2"), ("stype", "<u2"), ("srel", "<u2"),
                         ("option", "<u4")])

    def lookup_subjects(self, reqs) -> list:
        """reqs: [(res_type_id, res_id, perm_slot, subj_type_id, subj_rel_slot, wildcard_option)] of this rank (subj_rel_slot
        = SREL_NONE for a plain subject type; wildcard_option ZG_WILDCARDS_INCLUDE = 0 or EXCLUDE = 1). -> per request
        (ids, wildcard, excluded): the ascending uint32 ids listed, whether the wildcard entry is present, and the
        ascending uint32 ids it excludes; None where zg_lookup_subjects on a replica returns ZG_EDEPTH."""
        mine = np.zeros(len(reqs), self.SUBJ_REQ)
        for i, (rt, res, perm, st, srel, opt) in enumerate(reqs):
            mine[i] = (res, rt, perm, st, srel, opt)
        every, home, first = self._gather_requests(mine)
        out = [None] * mine.size
        for lo in range(0, every.size, LOOKUP_ROUND):
            self._subjects_round(every[lo:lo + LOOKUP_ROUND], home[lo:lo + LOOKUP_ROUND], lo - first, out)
        return out

    def _subjects_round(self, reqs, home, base, out):
        """One round of <= 64 lookups on every rank; answers of this rank's lookups go to out[base + k]."""
        t, w, dev, e = self.t, self.t.world, self.t.device, self.e
        K = reqs.size
        self.stats["rounds"] += 1
        protos = np.zeros(K, CHECK_DTYPE)
        protos["res"], protos["perm"], protos["stype"], protos["srel"] = reqs["res"], reqs["perm"], reqs["stype"], reqs["srel"]
        front = torch.empty(self.walk_cap * 8, dtype=torch.uint8, device=dev)
        routed = torch.empty(self.walk_cap * 8, dtype=torch.uint8, device=dev)
        n_front = e.shard_subjects_begin_dev(reqs["res_type"], protos, reqs["option"], home, self.walk_cap, front.data_ptr())
        self.stats["admitted"] += n_front
        level, overflow = 0, False
        while True:
            # levels 0 .. MAX_DEPTH + 1 are expanded, as on a replica; one more exchange reports the last admissions'
            # overflow and ends the walk
            live = n_front if level <= MAX_DEPTH + 1 else 0
            sc, ovf = e.shard_subjects_expand_dev(front.data_ptr(), live, w, routed.data_ptr())
            got = t.exchange_counts([c << 2 | (live > 0) << 1 | int(ovf) for c in sc])
            if any(g & 1 for g in got):
                overflow = True
                break
            if not any(g & 2 for g in got):  # no rank had a frontier at this level: the walk is over
                break
            self.stats["levels"] += 1
            rc = [g >> 2 for g in got]
            arrived = t.alltoall(routed[: sum(sc) * 8], sc, rc, 8)
            self.stats["entries_sent"] += sum(sc) - sc[t.rank]
            self.stats["bytes_sent"] += (sum(sc) - sc[t.rank]) * 8
            n_front = e.shard_subjects_admit_dev(arrived.data_ptr() if sum(rc) else 0, sum(rc), front.data_ptr())
            self.stats["admitted"] += n_front
            level += 1
        if overflow and K > 1:
            self.stats["halvings"] += 1
            h = K // 2
            self._subjects_round(reqs[:h], home[:h], base, out)
            self._subjects_round(reqs[h:], home[h:], base + h, out)
            return
        if overflow:
            self.stats["fallbacks"] += 1
        need = e.shard_subjects_candidates_dev(overflow, 0, 0)
        item = DeviceShardedChecker.ITEM
        items = torch.empty(max(need, 1) * item, dtype=torch.uint8, device=dev)
        n = e.shard_subjects_candidates_dev(overflow, items.data_ptr(), need)
        self.stats["candidates"] += n
        codes = self._verify(items, n)
        granted, failed = e.shard_subjects_verdicts_dev(codes.data_ptr() if n else 0, n)
        # the probe verdicts are known on the resources' owners only: every rank ORs every rank's masks
        masks = np.array([granted, failed], dtype=np.uint64).view(np.uint8)
        got = t.alltoall(torch.from_numpy(np.tile(masks, w)).to(dev), [1] * w, [1] * w, 16)
        got = np.bitwise_or.reduce(got.cpu().numpy().view(np.uint64).reshape(w, 2), axis=0)
        granted, failed = int(got[0]), int(got[1])
        self.stats["bytes_sent"] += 16 * (w - 1)
        nw_items = torch.empty(max(n, 1) * item, dtype=torch.uint8, device=dev)
        n_nw = e.shard_subjects_nowild_dev(codes.data_ptr() if n else 0, n, granted, failed, nw_items.data_ptr(), max(n, 1))
        self.stats["nowild_verified"] += n_nw
        # every rank takes part in the no-wildcards verification when any lookup of the round is granted
        nw_codes = self._verify(nw_items, n_nw, no_wildcards=True) if granted & ~failed else nw_items[:1]
        keys = torch.empty(max(n, 1) * 8, dtype=torch.uint8, device=dev)
        sc = e.shard_subjects_route_dev(nw_codes.data_ptr() if n_nw else 0, n_nw, w, keys.data_ptr())
        rc = t.exchange_counts(sc)
        arrived = t.alltoall(keys[: sum(sc) * 8], sc, rc, 8)
        self.stats["bytes_sent"] += (sum(sc) - sc[t.rank]) * 8
        nk = sum(rc)
        ids = torch.empty(max(nk, 1) * 4, dtype=torch.uint8, device=dev)
        listed, excluded = e.shard_subjects_finish_dev(arrived.data_ptr() if nk else 0, nk, ids.data_ptr(), K)
        host = ids[: nk * 4].cpu().numpy().view(np.uint32)
        at_l, at_x = 0, sum(listed)
        for k in range(K):
            if home[k] == t.rank:
                wild = bool((granted >> k) & 1) and reqs["option"][k] == WILDCARDS_INCLUDE
                out[base + k] = None if (failed >> k) & 1 else (
                    host[at_l:at_l + listed[k]].copy(), wild, host[at_x:at_x + excluded[k]].copy())
            at_l += listed[k]
            at_x += excluded[k]
