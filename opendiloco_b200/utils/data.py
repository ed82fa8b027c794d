"""Data pipeline: synthetic tokens (fast path), HF streaming text (when a tokenizer/dataset is reachable), collation.

Reference behaviour being reproduced (SURVEY.md E7, Appendix A):
  * ``FakeTokenizedDataset``: infinite random token ids in [3, vocab), attention mask all ones (utils.py:155-167),
    used with TEST_VOCAB_SIZE=1024 (train_fsdp.py:66,133-134);
  * causal-LM collation: labels = input_ids with pad positions -> -100 (DataCollatorForLanguageModeling(mlm=False));
  * worker-major sharding: rank = world_rank * world_size + local_rank of galaxy_size * world_size
    (train_fsdp.py:151-156);
  * resumable loader state (torchdata StatefulDataLoader: train_fsdp.py:163-168, ckpt_utils.py:83-87).

``SyntheticTokenLoader`` is the GPU-side fast path: batches are produced directly as pinned [B, S] int64 tensors
(by the C++ prefetcher in ``libodbhost.so`` when built) so the H2D copy is a single async DMA per micro-batch.
"""
from __future__ import annotations

from typing import Any, Generator, Iterator

import os

import torch
from torch.utils.data import IterableDataset

TEST_VOCAB_SIZE = 1024
IGNORE_INDEX = -100


class FakeTokenizedDataset(IterableDataset):
    """Infinite random sequences of length ``seq_len`` over ``[3, vocab_size)`` (reference utils.py:155-167).
    ``seed`` (an extension) makes the stream reproducible per rank; None keeps the reference's unseeded behaviour."""

    def __init__(self, seq_len: int, vocab_size: int, seed: int | None = None):
        assert vocab_size > 3, "Vocab size must be greater than 3"
        self.seq_len, self.vocab_size, self.seed = seq_len, vocab_size, seed

    def __iter__(self) -> Generator[dict[str, Any], Any, None]:
        gen = None
        if self.seed is not None:
            gen = torch.Generator().manual_seed(self.seed)
        while True:
            ids = torch.randint(3, self.vocab_size, (self.seq_len,), generator=gen).tolist()
            yield {"input_ids": ids, "attention_mask": [1] * self.seq_len}


def collate_causal_lm(features: list[dict], pad_token_id: int | None = None) -> dict[str, torch.Tensor]:
    """Pad to the longest sequence in the batch and build labels (pad -> -100)."""
    mx = max(len(f["input_ids"]) for f in features)
    pad = pad_token_id if pad_token_id is not None else 0
    ids = torch.full((len(features), mx), pad, dtype=torch.int64)
    mask = torch.zeros((len(features), mx), dtype=torch.int64)
    for i, f in enumerate(features):
        n = len(f["input_ids"])
        ids[i, :n] = torch.as_tensor(f["input_ids"], dtype=torch.int64)
        m = f.get("attention_mask")
        mask[i, :n] = torch.as_tensor(m, dtype=torch.int64) if m is not None else 1
    labels = ids.clone()
    labels[mask == 0] = IGNORE_INDEX
    if pad_token_id is not None:
        labels[ids == pad_token_id] = IGNORE_INDEX
    return {"input_ids": ids, "attention_mask": mask, "labels": labels}


class SyntheticTokenLoader:
    """Resumable iterator of pinned synthetic batches ``{"input_ids", "attention_mask", "labels"}`` of shape [B, S].

    Token law = the reference fake data (uniform over [3, vocab)); the generator is seeded per (seed, rank) and its
    state is part of ``state_dict()`` so checkpoint/resume reproduces the stream exactly."""

    def __init__(self, batch_size: int, seq_len: int, vocab_size: int = TEST_VOCAB_SIZE, seed: int = 0, rank: int = 0,
                 pin_memory: bool | None = None, with_mask: bool = True):
        self.batch_size, self.seq_len, self.vocab_size = batch_size, seq_len, vocab_size
        self.gen = torch.Generator().manual_seed(seed * 1_000_003 + rank)
        self.pin = torch.cuda.is_available() if pin_memory is None else pin_memory
        self.with_mask = with_mask
        self._mask = torch.ones(batch_size, seq_len, dtype=torch.int64)
        self.batches_yielded = 0

    def __iter__(self) -> Iterator[dict[str, torch.Tensor]]:
        return self

    def __next__(self) -> dict[str, torch.Tensor]:
        ids = torch.empty(self.batch_size, self.seq_len, dtype=torch.int64, pin_memory=self.pin)
        torch.randint(3, self.vocab_size, ids.shape, generator=self.gen, out=ids)
        self.batches_yielded += 1
        out = {"input_ids": ids, "labels": ids}
        if self.with_mask:
            out["attention_mask"] = self._mask
        return out

    def state_dict(self) -> dict:
        return {"rng": self.gen.get_state(), "batches_yielded": self.batches_yielded}

    def load_state_dict(self, sd: dict) -> None:
        self.gen.set_state(sd["rng"])
        self.batches_yielded = int(sd["batches_yielded"])


class _RingLoader:
    """Consumer side of the C++ prefetch ring (``csrc/host/prefetch_ring.h``): a background thread keeps a ring of PINNED
    [B, S] int64 buffers filled, ``next()`` is a pointer hand-off and the H2D copy is the only per-batch host work.  A
    stream is a pure function of the batch index, so ``state_dict`` is one integer."""

    def __init__(self, batch_size: int, seq_len: int, nbuf: int, pin_memory: bool | None):
        import ctypes

        from .. import _lib

        lib = _lib.host_lib()
        if lib is None or not hasattr(lib, "odb_tg_create"):
            raise RuntimeError("libodbhost.so is not built (python -m opendiloco_b200.build)")
        self._ct, self._lib = ctypes, lib
        lib.odb_tg_create.restype = ctypes.c_void_p
        lib.odb_tg_create.argtypes = [ctypes.c_uint64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int,
                                      ctypes.POINTER(ctypes.c_void_p), ctypes.c_int64]
        lib.odb_tg_next.argtypes = [ctypes.c_void_p]
        lib.odb_tg_release.argtypes = [ctypes.c_void_p, ctypes.c_int]
        lib.odb_tg_position.argtypes = [ctypes.c_void_p]
        lib.odb_tg_position.restype = ctypes.c_int64
        lib.odb_tg_destroy.argtypes = [ctypes.c_void_p]
        pin = torch.cuda.is_available() if pin_memory is None else pin_memory
        self.batch_size, self.seq_len = batch_size, seq_len
        self.bufs = [torch.empty(batch_size, seq_len, dtype=torch.int64, pin_memory=pin) for _ in range(nbuf)]
        self._h = None
        self._held: int | None = None
        self._inflight: list = []          # (slot, cuda event) pairs whose H2D copy may still be running

    def _buf_array(self):
        return (self._ct.c_void_p * len(self.bufs))(*[b.data_ptr() for b in self.bufs])

    def _start(self, batch_index: int) -> None:        # pragma: no cover - provided by the subclasses
        raise NotImplementedError

    def __iter__(self):
        return self

    def __next__(self) -> dict[str, torch.Tensor]:
        # The consumer enqueues its (async) H2D copy of a batch before asking for the next one, so an event recorded
        # NOW on the current stream covers the copy of the previously handed-out slot.  A slot goes back to the
        # prefetch thread only after that event completed: the CPU may run up to nbuf-2 micro-batches ahead of the GPU.
        if self._held is not None:
            ev = None
            if torch.cuda.is_available() and self.bufs[0].is_pinned():
                ev = torch.cuda.Event()
                ev.record()
            self._inflight.append((self._held, ev))
        while len(self._inflight) > len(self.bufs) - 2:
            slot, ev = self._inflight.pop(0)
            if ev is not None:
                ev.synchronize()
            self._lib.odb_tg_release(self._h, slot)
        slot = self._lib.odb_tg_next(self._h)
        self._held = slot
        ids = self.bufs[slot]
        return {"input_ids": ids, "labels": ids}

    def state_dict(self) -> dict:
        pos = self._lib.odb_tg_position(self._h)
        return {"batches_yielded": int(pos)}

    def load_state_dict(self, sd: dict) -> None:
        self.close()
        self._held = None
        self._inflight = []
        self._start(int(sd["batches_yielded"]))

    def close(self) -> None:
        if self._h is not None:
            self._lib.odb_tg_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class NativeTokenLoader(_RingLoader):
    """SyntheticTokenLoader backed by the C++ prefetcher (``csrc/host/tokengen.cc``): uniform tokens in [3, vocab), a
    pure function of (seed, rank, batch index)."""

    def __init__(self, batch_size: int, seq_len: int, vocab_size: int = TEST_VOCAB_SIZE, seed: int = 0, rank: int = 0,
                 nbuf: int = 8, pin_memory: bool | None = None):
        super().__init__(batch_size, seq_len, nbuf, pin_memory)
        self.vocab_size = vocab_size
        self.seed = (seed * 1_000_003 + rank) & 0xFFFFFFFFFFFFFFFF
        self._start(0)

    def _start(self, batch_index: int) -> None:
        self._h = self._lib.odb_tg_create(self.seed, 3, self.vocab_size, self.batch_size * self.seq_len, len(self.bufs),
                                          self._buf_array(), batch_index)


TOKEN_SHARD_MAGIC = b"ODBTOK1\0"


def write_token_shard(path: str, tokens, bytes_per_token: int | None = None) -> None:
    """Write a 1-D token array as one shard of the pre-tokenised corpus format (32-byte header + uint16 / uint32 tokens;
    ``csrc/host/tokenfile.cc``).  uint16 is chosen automatically when every token fits."""
    import ctypes

    from .. import _lib

    t = torch.as_tensor(tokens, dtype=torch.int64).contiguous().view(-1)
    if bytes_per_token is None:
        bytes_per_token = 2 if (t.numel() == 0 or int(t.max()) <= 0xFFFF) else 4
    lib = _lib.host_lib()
    if lib is None or not hasattr(lib, "odb_tf_write"):
        raise RuntimeError("libodbhost.so is not built (python -m opendiloco_b200.build)")
    lib.odb_tf_write.argtypes = [ctypes.c_char_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int]
    rc = lib.odb_tf_write(str(path).encode(), t.data_ptr(), t.numel(), int(bytes_per_token))
    if rc != 0:
        raise OSError(f"could not write token shard {path} (code {rc}: token out of range for {bytes_per_token}-byte storage?)")


class TokenFileLoader(_RingLoader):
    """Causal-LM batches straight from pre-tokenised shards (``csrc/host/tokenfile.cc``): mmap + prefetch thread, windows
    of ``seq_len`` tokens, seeded shuffle that visits every window once per epoch, disjoint samples per rank.  Feeds the
    ~6 M tokens/s an 8-GPU box consumes, which on-the-fly tokenisation (the reference's pipeline) cannot.

    ``paths``: shard files, or one glob pattern.  Shards come from ``write_token_shard`` / ``scripts/tokenize_corpus.py``;
    header-less ``.bin`` files of uint16 / uint32 tokens work with ``raw_bytes_per_token``."""

    def __init__(self, paths, batch_size: int, seq_len: int, rank: int = 0, world: int = 1, seed: int = 0, shuffle: bool = True,
                 nbuf: int = 8, pin_memory: bool | None = None, raw_bytes_per_token: int = 2):
        import glob as _glob

        super().__init__(batch_size, seq_len, nbuf, pin_memory)
        if isinstance(paths, (str, os.PathLike)):
            found = sorted(_glob.glob(str(paths)))
            paths = found if found else [str(paths)]
        self.paths = [str(p) for p in paths]
        self.rank, self.world, self.seed, self.shuffle, self.raw_bytes = rank, world, seed, shuffle, raw_bytes_per_token
        ct = self._ct
        self._lib.odb_tf_open.restype = ct.c_void_p
        self._lib.odb_tf_open.argtypes = [ct.POINTER(ct.c_char_p), ct.c_int, ct.c_int, ct.c_int64, ct.c_int64, ct.c_int64, ct.c_int64,
                                          ct.c_uint64, ct.c_int, ct.c_int, ct.POINTER(ct.c_void_p), ct.c_int64, ct.POINTER(ct.c_int64)]
        self.windows_per_epoch = 0
        self._start(0)

    def _start(self, batch_index: int) -> None:
        ct = self._ct
        arr = (ct.c_char_p * len(self.paths))(*[p.encode() for p in self.paths])
        windows = ct.c_int64(0)
        self._h = self._lib.odb_tf_open(arr, len(self.paths), self.raw_bytes, self.seq_len, self.batch_size, self.rank, self.world,
                                        self.seed & 0xFFFFFFFFFFFFFFFF, int(self.shuffle), len(self.bufs), self._buf_array(),
                                        batch_index, ct.byref(windows))
        self.windows_per_epoch = int(windows.value)
        if not self._h:
            raise ValueError(f"could not open token shards {self.paths[:3]}...: unreadable file, or fewer than "
                             f"batch_size * world = {self.batch_size * self.world} windows of {self.seq_len} tokens "
                             f"({self.windows_per_epoch} found)")

    @property
    def batches_per_epoch(self) -> int:
        return self.windows_per_epoch // (self.batch_size * self.world)


def data_rank(world_rank: int | None, galaxy_size: int | None, world_size: int, rank: int, local_rank: int) -> tuple[int, int]:
    """(shard index, number of shards) with the reference's worker-major rule (train_fsdp.py:151-156)."""
    if galaxy_size is not None and world_rank is not None:
        return world_rank * world_size + local_rank, galaxy_size * world_size
    return rank, world_size


def get_text_dataloader(dataset_name_or_path: str, tokenizer_name: str, seq_length: int, batch_size: int, shard: int,
                        num_shards: int, num_workers: int = 4, pad_to_max: bool = True, c4_tiny: bool = False,
                        seed: int | None = None, split: str = "train"):
    """Streaming text -> tokens -> causal-LM batches (reference get_dataloader, train_fsdp.py:132-168;
    train_diloco_torch.py:201-229).  Needs ``datasets`` + a locally available tokenizer/dataset (no network here)."""
    from datasets import load_dataset
    from datasets.distributed import split_dataset_by_node
    from transformers import AutoTokenizer

    try:
        from torchdata.stateful_dataloader import StatefulDataLoader as Loader
    except Exception:  # pragma: no cover
        from torch.utils.data import DataLoader as Loader

    tok = AutoTokenizer.from_pretrained(tokenizer_name, use_fast=True)
    tok.pad_token = "</s>"
    if c4_tiny:
        ds = load_dataset("PrimeIntellect/c4-tiny", "en")
    else:
        ds = load_dataset(dataset_name_or_path, "en", streaming=True)
    if seed is not None:
        ds = ds.shuffle(seed=seed)

    def tokenize(batch):
        kw = dict(truncation=True, max_length=seq_length)
        if pad_to_max:
            kw["padding"] = "max_length"
        return tok(batch["text"], **kw)

    cols = [c for c in ("text", "timestamp", "url") if c in (ds[split].column_names or ["text", "timestamp", "url"])]
    tokenized = ds.map(tokenize, batched=True, remove_columns=cols)[split]
    sharded = split_dataset_by_node(tokenized, world_size=num_shards, rank=shard)
    pad_id = tok.pad_token_id

    def collate(features):
        return collate_causal_lm(features, pad_id)

    return Loader(sharded, collate_fn=collate, batch_size=batch_size, num_workers=num_workers)


def get_fake_dataloader(seq_length: int, batch_size: int, vocab_size: int = TEST_VOCAB_SIZE, num_workers: int = 0,
                        seed: int | None = None):
    """The reference's --fake-data loader: FakeTokenizedDataset through a (stateful) torch DataLoader."""
    try:
        from torchdata.stateful_dataloader import StatefulDataLoader as Loader
    except Exception:  # pragma: no cover
        from torch.utils.data import DataLoader as Loader
    return Loader(FakeTokenizedDataset(seq_length, vocab_size, seed), collate_fn=collate_causal_lm, batch_size=batch_size,
                  num_workers=num_workers)
