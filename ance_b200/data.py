"""Token-cache I/O of the ANN refresh: the reference's dataset surface plus a bulk reader.

Drop-in for the reference's
  * ``EmbeddingCache``     utils/util.py:257-307  (fixed-record binary token store)
  * ``StreamingDataset``   utils/util.py:310-329  (rank-strided IterableDataset)
  * ``GetProcessingFn``    data/msmarco_data.py:275-303 and data/DPR_data.py:276-296
with the same names, argument meaning and error behaviour, so the trainer (which random-accesses
the same caches, data/msmarco_data.py:348-358) and any code written against the reference keep
working.  ``StridedBatchReader`` is what the GPU refresher itself uses: it memory-maps the file
once, takes this rank's ``i % world_size == rank`` records with numpy (no per-record Python), and
yields pinned ``(ids int32[B,L], lens int32[B], idx int64[B])`` batches; the attention mask is
built on the GPU from ``lens`` (or from ``ids != 0`` for DPR).

Record layout (SURVEY.md Appendix B): 4-byte BIG-endian length, then L native int32 token ids.
"""
from __future__ import annotations

import json
from typing import Iterator, Optional, Tuple

import numpy as np
import torch
import torch.distributed as dist
from torch.utils.data import IterableDataset, TensorDataset


class EmbeddingCache:
    """Fixed-record token store with the reference class's public surface (utils/util.py:257-307: attributes `dtype`,
    `total_number`, `record_size`, `ix_array`; `open` / `close` / context manager; `cache[i] -> (length, ids[L])`; iteration
    in `ix_array` order; `len`; `read_single_record`), implemented over ONE read-only memory map of the file instead of a
    seek pointer: records are views into the mapping (zero-copy, page-cache backed), random access needs no syscall, and the
    object is safe to share between threads and across `fork` (the reference's shared file position is why it must run with
    `num_workers=0`, SURVEY.md par. 8b).  Opening is lazy: `with cache:` / `cache.open()` keep working but are not required."""

    def __init__(self, base_path, seed=-1):
        self.base_path = base_path
        with open(base_path + "_meta", "r") as f:
            meta = json.load(f)
        self.dtype = np.dtype(meta["type"])
        self.total_number = int(meta["total_number"])
        self._tokens = int(meta["embedding_size"])
        self.record_size = self._tokens * self.dtype.itemsize + 4          # 4-byte big-endian length + the ids
        # visiting order of __iter__: a seeded permutation (the trainer's shuffled passes) or file order
        self.ix_array = (np.random.RandomState(seed).permutation(self.total_number) if seed >= 0
                         else np.arange(self.total_number))
        self._map = None
        self._cursor = 0         # next record of read_single_record()

    # -- mapping --------------------------------------------------------------------------------
    @property
    def embedding_size(self) -> int:
        return self._tokens

    def memmap(self) -> np.ndarray:
        """The whole file as a structured array: field 'len' (>i4) and 'ids' (dtype[L])."""
        if self._map is None:
            rec = np.dtype([("len", ">i4"), ("ids", self.dtype, (self._tokens,))])
            self._map = (np.zeros((0,), dtype=rec) if self.total_number == 0
                         else np.memmap(self.base_path, dtype=rec, mode="r", shape=(self.total_number,)))
        return self._map

    def open(self):
        self.memmap()
        self._cursor = 0

    def close(self):
        self._map = None

    def __enter__(self):
        self.open()
        return self

    def __exit__(self, exc_type, exc, tb):
        self.close()

    # -- record access --------------------------------------------------------------------------
    def _record(self, i: int):
        r = self.memmap()[i]
        return int(r["len"]), np.asarray(r["ids"])

    def read_single_record(self):
        """The record at the cursor (set by `open()` / `cache[i]`), then advance — the reference's sequential read."""
        if self._cursor >= self.total_number:
            return 0, np.empty((0,), dtype=self.dtype)       # what reading past the end of the file yields upstream
        rec = self._record(self._cursor)
        self._cursor += 1
        return rec

    def __getitem__(self, key):
        # (the reference's own check is `key > total_number`, util.py:293: record `total_number` then fails later on an
        # empty buffer; here the bound is exact and the message is the reference's)
        if key < 0 or key >= self.total_number:
            raise IndexError(
                "Index {} is out of bound for cached embeddings of size {}".format(key, self.total_number))
        self._cursor = int(key) + 1
        return self._record(int(key))

    def __iter__(self):
        for i in self.ix_array:
            yield self[int(i)]

    def __len__(self):
        return self.total_number


class StreamingDataset(IterableDataset):
    """Rank-strided stream with the reference's contract (utils/util.py:310-329): element i belongs to rank
    `i % world_size` when a process group is initialised (every element otherwise, or with distributed=False), and each
    kept element expands to the records `fn(element, i)` returns."""

    def __init__(self, elements, fn, distributed=True):
        super().__init__()
        self.elements = elements
        self.fn = fn
        self.distributed = distributed
        self.num_replicas = -1       # filled in at iteration time, as upstream (-1: no process group)
        self.rank = 0

    def _mine(self, i: int) -> bool:
        return not self.distributed or self.num_replicas == -1 or i % self.num_replicas == self.rank

    def __iter__(self):
        if dist.is_available() and dist.is_initialized():
            self.num_replicas, self.rank = dist.get_world_size(), dist.get_rank()
        for i, element in enumerate(self.elements):
            if self._mine(i):
                yield from self.fn(element, i)


def GetProcessingFn(args, query=False):
    """data/msmarco_data.py:275-303: record -> [(input_ids int32[L], attention_mask bool[L],
    token_type_ids uint8[L], idx int64)]."""

    def fn(vals, i):
        passage_len, passage = vals
        max_len = args.max_query_length if query else args.max_seq_length
        pad_len = max(0, max_len - passage_len)
        token_type_ids = ([0] if query else [1]) * passage_len + [0] * pad_len
        attention_mask = [1] * passage_len + [0] * pad_len
        dataset = TensorDataset(
            torch.tensor(np.asarray(passage)[None, :], dtype=torch.int),
            torch.tensor([attention_mask], dtype=torch.bool),
            torch.tensor([token_type_ids], dtype=torch.uint8),
            torch.tensor([i], dtype=torch.long))
        return [ts for ts in dataset]

    return fn


def _parse_ann_line(line: str):
    """`qid \\t pos_pid \\t neg,neg,...` -- the line grammar of ann_training_data_N (run_ann_data_gen.py:326-334)."""
    a = line.split("\t")
    return int(a[0]), int(a[1]), [int(x) for x in a[2].split(",")]


def GetTrainingDataProcessingFn(args, query_cache, passage_cache):
    """data/msmarco_data.py:306-334 (the trainer's side of the refresh protocol): one ANN line -> for every negative a
    (query, positive, label 1) and a (query, negative, label 0) record."""
    qfn, pfn = GetProcessingFn(args, query=True), GetProcessingFn(args, query=False)

    def fn(line, i):
        qid, pos_pid, neg_pids = _parse_ann_line(line)
        q = qfn(query_cache[qid], qid)[0]
        pos = pfn(passage_cache[pos_pid], pos_pid)[0]
        pos_label, neg_label = torch.tensor(1, dtype=torch.long), torch.tensor(0, dtype=torch.long)
        for neg_pid in neg_pids:
            neg = pfn(passage_cache[neg_pid], neg_pid)[0]
            yield (q[0], q[1], q[2], pos[0], pos[1], pos[2], pos_label)
            yield (q[0], q[1], q[2], neg[0], neg[1], neg[2], neg_label)

    return fn


def GetTripletTrainingDataProcessingFn(args, query_cache, passage_cache):
    """data/msmarco_data.py:337-362: one ANN line -> one (query, positive, negative) triplet per negative, the records
    `run_ann.py:240-292` feeds to `model(*batch)`."""
    qfn, pfn = GetProcessingFn(args, query=True), GetProcessingFn(args, query=False)

    def fn(line, i):
        qid, pos_pid, neg_pids = _parse_ann_line(line)
        q = qfn(query_cache[qid], qid)[0]
        pos = pfn(passage_cache[pos_pid], pos_pid)[0]
        for neg_pid in neg_pids:
            neg = pfn(passage_cache[neg_pid], neg_pid)[0]
            yield (q[0], q[1], q[2], pos[0], pos[1], pos[2], neg[0], neg[1], neg[2])

    return fn


class TripletBatchReader:
    """Bulk form of `StreamingDataset(lines, GetTripletTrainingDataProcessingFn(...))` + DataLoader(batch_size): the
    triplets of this rank's ANN lines (line i -> rank i % world_size, utils/util.py:321-323), in the same order, as
    pinned int32 id matrices and int32 lengths -- token rows come from the caches' memmaps in one vectorised gather per
    batch instead of one 3-tensor TensorDataset per record.  Yields (q_ids, q_len, pos_ids, pos_len, neg_ids, neg_len)."""

    def __init__(self, lines, query_cache: "EmbeddingCache", passage_cache: "EmbeddingCache", batch_size: int,
                 max_query_length: int, max_seq_length: int, rank: int = 0, world_size: int = 1, pin: bool = True):
        self.lines, self.qc, self.pc = lines, query_cache, passage_cache
        self.batch_size, self.rank, self.world = int(batch_size), int(rank), int(world_size)
        self.lq, self.lp = int(max_query_length), int(max_seq_length)
        self.pin = pin and torch.cuda.is_available()

    def _triplets(self):
        for i, line in enumerate(self.lines):
            if i % self.world != self.rank:
                continue
            qid, pos, negs = _parse_ann_line(line)
            for n in negs:
                yield qid, pos, n

    @staticmethod
    def _gather(mm, rows, L):
        rec = mm[np.asarray(rows, dtype=np.int64)]
        lens = rec["len"].astype(np.int32)
        ids = np.ascontiguousarray(rec["ids"][:, :L]).astype(np.int32)
        return ids, np.minimum(lens, L)

    def __iter__(self):
        qmm, pmm = self.qc.memmap(), self.pc.memmap()
        buf = []

        def emit(chunk):
            cols = list(zip(*chunk))
            out = []
            for mm, rows, L in ((qmm, cols[0], self.lq), (pmm, cols[1], self.lp), (pmm, cols[2], self.lp)):
                ids, lens = self._gather(mm, rows, L)
                ti, tl = torch.from_numpy(ids), torch.from_numpy(lens)
                out += [ti.pin_memory() if self.pin else ti, tl.pin_memory() if self.pin else tl]
            return tuple(out)

        for t in self._triplets():
            buf.append(t)
            if len(buf) == self.batch_size:
                yield emit(buf)
                buf = []
        if buf:
            yield emit(buf)


def GetProcessingFnDPR(args, query=False):
    """data/DPR_data.py:276-296: as above but attention_mask = ids != 0 and token types all 0."""

    def fn(vals, i):
        passage_len, passage = vals
        passage = np.asarray(passage)
        dataset = TensorDataset(
            torch.tensor(passage[None, :], dtype=torch.int),
            torch.tensor((passage != 0)[None, :], dtype=torch.bool),
            torch.zeros((1, passage.shape[0]), dtype=torch.uint8),
            torch.tensor([i], dtype=torch.long))
        return [ts for ts in dataset]

    return fn


class StridedBatchReader:
    """Bulk, rank-strided batches of one token cache.

    Yields ``(ids, lens, idx)`` with exactly the records, order and batch boundaries the
    reference's ``DataLoader(StreamingDataset(cache, fn), batch_size=B)`` produces on this rank
    (run_ann_data_gen.py:199-202): records ``rank, rank+W, rank+2W, ...`` in groups of B, last
    batch ragged.  Tensors are pinned when CUDA is available so the H2D copy can be asynchronous.
    """

    def __init__(self, cache: EmbeddingCache, batch_size: int, rank: int = 0, world_size: int = 1,
                 max_len: Optional[int] = None, pin: Optional[bool] = None):
        if batch_size <= 0:
            raise ValueError("batch_size must be positive")
        self.cache = cache
        self.batch_size = int(batch_size)
        self.rank, self.world_size = int(rank), int(world_size)
        self.L = cache.embedding_size
        if max_len is not None and max_len != self.L:
            raise ValueError(f"cache records hold {self.L} tokens but max length {max_len} was requested")
        self.pin = torch.cuda.is_available() if pin is None else pin
        self.n_local = len(range(self.rank, cache.total_number, self.world_size))

    def __len__(self) -> int:
        return (self.n_local + self.batch_size - 1) // self.batch_size

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
        mm = self.cache.memmap()
        n, W, B = self.cache.total_number, self.world_size, self.batch_size
        for b0 in range(0, self.n_local, B):
            first = self.rank + b0 * W
            stop = min(n, self.rank + (b0 + B) * W)
            idx = np.arange(first, stop, W, dtype=np.int64)
            recs = mm[first:stop:W]
            ids = torch.from_numpy(np.array(recs["ids"], dtype=np.int32, order="C"))
            lens = torch.from_numpy(np.array(recs["len"]).astype(np.int32))
            idx_t = torch.from_numpy(idx)
            if self.pin:
                ids, lens = ids.pin_memory(), lens.pin_memory()
            yield ids, lens, idx_t


class AnnDataWatcher:
    """The trainer's in-process hot swap of ANN training data (drivers/run_ann.py:182-228), as one object.

    The reference's training loop polls `get_latest_ann_data(args.ann_dir)` every `logging_steps`, and when the refresher has
    published a new `ann_ndcg_N` it re-reads `ann_training_data_N`, truncates it to a multiple of the world size
    (`aligned_size`, run_ann.py:193-195), rebuilds its streaming dataset and restarts the iterator.  `poll()` does exactly
    that and returns None when nothing new is there, else a `Swap` with the reference's bookkeeping values (`ann_no`,
    `dev_ndcg`, `checkpoint`, `checkpoint_no`, number of lines) and a fresh `TripletBatchReader` over the new lines for this
    rank.  It only ever sees complete files: the refresher publishes `ann_training_data_N` first and `ann_ndcg_N` last, both
    through an atomic rename (ance_b200/postprocess.py)."""

    class Swap:
        def __init__(self, ann_no, ann_path, ndcg_json, lines, reader):
            self.ann_no, self.ann_path, self.lines, self.reader = ann_no, ann_path, lines, reader
            self.dev_ndcg = ndcg_json.get("ndcg")
            self.checkpoint = ndcg_json.get("checkpoint")
            import re
            nums = re.findall(r"\d+", self.checkpoint or "")
            self.checkpoint_no = int(nums[-1]) if nums else 0      # utils/util.py:224-226

    def __init__(self, ann_dir: str, query_cache: "EmbeddingCache", passage_cache: "EmbeddingCache", batch_size: int,
                 max_query_length: int, max_seq_length: int, rank: int = 0, world_size: int = 1, pin: bool = True):
        self.ann_dir, self.qc, self.pc = ann_dir, query_cache, passage_cache
        self.batch_size, self.lq, self.lp = batch_size, max_query_length, max_seq_length
        self.rank, self.world, self.pin = rank, world_size, pin
        self.last_ann_no = -1

    def poll(self):
        from .drivers.run_ann_data_gen import get_latest_ann_data
        ann_no, ann_path, ndcg_json = get_latest_ann_data(self.ann_dir)
        if ann_path is None or ann_no == self.last_ann_no:
            return None
        with open(ann_path, "r") as f:
            lines = f.readlines()
        lines = lines[:(len(lines) // self.world) * self.world]         # aligned_size
        reader = TripletBatchReader(lines, self.qc, self.pc, self.batch_size, self.lq, self.lp, rank=self.rank,
                                    world_size=self.world, pin=self.pin)
        self.last_ann_no = ann_no
        return AnnDataWatcher.Swap(ann_no, ann_path, ndcg_json, lines, reader)
