"""Host-side wrapper of the Dual-AR engine handle (fsb_lm_*).  PyTorch is used only for device memory
(weights, index tensors) and streams; all compute happens in libfishb200.so."""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib

STEP_ROWS = 32  # row tile of the decode step GEMM for engines of up to 32 slots
MAX_DECODE_BATCH = 64  # sequences per engine: above 32 the decode step runs its 64-row tile


def decode_row_tile(max_batch: int) -> int:
    """Rows of the decode step's GEMM tile and decode-state buffers for an engine of `max_batch` slots: 32 up to
    32 slots, 64 above. A sequence's bits do not depend on it (include/fishb200.h, fsb_lm_config.max_batch)."""
    return STEP_ROWS if max_batch <= STEP_ROWS else MAX_DECODE_BATCH


class _DevView:
    """Expose a raw device pointer through __cuda_array_interface__ so torch can view it (zero copy)."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {
            "shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 3, "strides": None,
        }


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def rope_table(seq_len: int, n_elem: int, base: float) -> torch.Tensor:
    """bf16 cos/sin table exactly as the reference builds it (llama.py:1004-1023): the table is an
    input of the kernels, so it is produced by the same torch ops the reference uses."""
    inv = 1.0 / (base ** (torch.arange(0, n_elem, 2)[: n_elem // 2].float() / n_elem))
    ang = torch.outer(torch.arange(seq_len), inv)
    cis = torch.polar(torch.ones_like(ang), ang)
    return torch.stack([cis.real, cis.imag], dim=-1).to(torch.bfloat16)


def interleave_w13(w1: torch.Tensor, w3: torch.Tensor) -> torch.Tensor:
    """Fused gate|up projection in the row order the step GEMM's SwiGLU epilogue expects (include/fishb200.h,
    d_w13): per 128-row tile t, rows 32w+l (l<16) = w1[64t+16w+l] and rows 32w+16+l = w3[64t+16w+l]; the
    hidden size is padded to a multiple of 64 with zero rows."""
    I, D = w1.shape
    Ip = (I + 63) // 64 * 64
    if Ip != I:
        pad = torch.zeros(Ip - I, D, dtype=w1.dtype, device=w1.device)
        w1, w3 = torch.cat([w1, pad]), torch.cat([w3, pad])
    g = w1.reshape(Ip // 16, 1, 16, D)
    u = w3.reshape(Ip // 16, 1, 16, D)
    return torch.cat([g, u], dim=1).reshape(2 * Ip, D).contiguous()


def bf16_round(v: float) -> float:
    """Sampling scalars are bf16 tensors in the reference (inference.py:303-304)."""
    return float(torch.tensor(v, dtype=torch.bfloat16).float())


KV_PAGE = 64  # positions per page of the slow KV cache (include/fishb200.h, fsb_lm_config.kv_pages)


def kv_pages_for(n_positions: int) -> int:
    return -(-int(n_positions) // KV_PAGE)


PREFIX_BLOCK = 16  # token rows per link of a cached prefix's hash chain (= LmEngine.MIN_REUSE)


def _chain_keys(rows: np.ndarray) -> list:
    """Chained hashes of the whole PREFIX_BLOCK-row blocks of token rows [n, C+1]: key j names rows [0, 16 (j + 1))."""
    keys, h = [], 0
    for a in range(0, rows.shape[0] - PREFIX_BLOCK + 1, PREFIX_BLOCK):
        h = hash((h, rows[a:a + PREFIX_BLOCK].tobytes()))
        keys.append(h)
    return keys


def _common_rows(a: np.ndarray, b: np.ndarray) -> int:
    """Length of the common prefix of two token-row arrays [n, C+1]."""
    n = min(len(a), len(b))
    diff = np.flatnonzero((a[:n] != b[:n]).any(axis=1))
    return int(diff[0]) if len(diff) else n


@dataclass(eq=False)
class CachedRow:
    """A prompt prefix kept in the page pool after its request left its slot (KvPagePool.insert): a page-table row
    outside every slot, like a parked request's, that holds references to the pages of positions [0, n)."""

    row: np.ndarray  # pages of positions [0, n); -1 past them
    rows: np.ndarray  # token rows [n, C+1] (int32) whose K/V those positions hold, as prefill wrote it
    n: int
    keys: list  # _chain_keys(rows)
    stamp: int = 0  # last insert or reuse (KvPagePool.tick)


class KvPagePool:
    """Host side of the paged slow KV cache: which pool page holds each 64-position block of each slot.

    `table[slot, j]` is the page of positions [64 j, 64 j + 64) of the slot, -1 when none is mapped. A page can be
    mapped by several slots (a shared prompt prefix); `ref[page]` counts them and a page returns to the free list when
    the count drops to 0. A slot is live (reserved for a request that may still write) or retired: a retired slot keeps
    its pages mapped, as a prefix later requests may reuse, until an allocation needs them; retired slots are then
    released least recently retired first, and `on_reclaim(slot)` lets the owner forget what the slot held. A row can
    also be detached: taken out of the table with its page references, for a request that is parked between two frames
    and continues later in whichever slot is idle then.

    With `prefix_cache`, a prompt prefix also outlives its slot: `insert` keeps the pages of a retiring slot's prompt
    as a cached row (CachedRow), `lookup` finds the longest cached prefix of a prompt, and a reservation short of pages
    drops cached rows least recently used first, after the retired slots. Cached rows hold only pages nobody else
    needs: `available()` counts the pages only they map as available.

    Device effects are callbacks, so that the rules can run without a GPU: `copy_page(src, dst, n)` copies positions
    [0, n) of a page, stream-ordered before the writes that follow."""

    def __init__(self, slots: int, pages_per_slot: int, n_pages: int, copy_page=None, on_reclaim=None,
                 prefix_cache: bool = False):
        if n_pages < 1:
            raise ValueError(f"kv_pages must be >= 1, got {n_pages}")
        self.slots, self.pages_per_slot, self.n_pages = slots, pages_per_slot, n_pages
        self.table = np.full((slots, pages_per_slot), -1, dtype=np.int32)
        self.ref = np.zeros(n_pages, dtype=np.int32)
        self.free = list(range(n_pages - 1, -1, -1))  # popped from the end: page 0 first
        self.retired: dict[int, None] = {s: None for s in range(slots)}  # insertion order = retirement order
        self.detached: list[np.ndarray] = []  # rows of parked requests: they keep their page references, in no slot
        self.copy_page = copy_page or (lambda src, dst, n: None)
        self.on_reclaim = on_reclaim or (lambda slot: None)
        self.dirty = True
        self.peak = 0
        self.prefix_cache = bool(prefix_cache)
        self.cached: dict[CachedRow, None] = {}  # least recently used first
        self._index: dict[int, set] = {}  # chain key -> cached rows whose keys include it
        self.held: set = set()  # cached rows that are donors of the admission being reserved: dropped last
        self.tick = 0
        self.hits = 0  # admissions that mapped a cached prefix
        self.evictions = 0  # cached rows dropped because a reservation was short of pages

    # ---- queries ------------------------------------------------------------------------------------------------
    def in_use(self) -> int:
        return self.n_pages - len(self.free)

    def available(self) -> int:
        """Pages a reservation can get: free ones plus those that only retired slots and cached rows map."""
        live = [s for s in range(self.slots) if s not in self.retired]
        pages = np.concatenate([self.table[live].ravel(), *self.detached])
        return self.n_pages - len(np.unique(pages[pages >= 0]))

    def row_pages(self, row: np.ndarray) -> tuple[int, int]:
        """(pages `row` maps, pages no other row maps) of a slot's row (`table[slot]`) or a detached one: what a
        request holds, and what it gives back to `available()` once it is retired or dropped."""
        pages = row[row >= 0]
        return len(pages), int(np.count_nonzero(self.ref[pages] == 1))

    # ---- mapping ------------------------------------------------------------------------------------------------
    def _unmap(self, slot: int, first: int):
        """Unmap pages first.. of `slot` (a row never maps one page twice)."""
        row = self.table[slot, first:]
        pages = row[row >= 0]
        if len(pages):
            row[:] = -1
            self.ref[pages] -= 1
            self.free.extend(pages[self.ref[pages] == 0].tolist())
            self.dirty = True

    def release(self, slot: int):
        """Unmap every page of `slot`."""
        self._unmap(slot, 0)

    def retire(self, slot: int):
        """`slot` will not write again until its next reservation; its pages stay mapped until needed."""
        self.retired.setdefault(slot, None)

    # ---- parked requests: a page-table row outside every slot -------------------------------------------------------
    def detach(self, slot: int) -> np.ndarray:
        """Take the live `slot`'s row out of the table, with its page references: the pages count as live in
        `available()` and no reservation reclaims them (only rows of retired slots are released), while the slot, now
        mapping nothing, is free for another request. Pages other slots map too stay shared. No K/V moves."""
        if slot in self.retired:
            raise ValueError(f"slot {slot} is retired: only a live slot's pages can be detached")
        row = self.table[slot].copy()
        self.table[slot] = -1
        self.detached.append(row)
        self.retired[slot] = None
        self.dirty = True
        return row

    def _undetach(self, row: np.ndarray):
        k = next((i for i, r in enumerate(self.detached) if r is row), None)
        if k is None:
            raise ValueError("not a detached row of this pool (or already attached / dropped)")
        del self.detached[k]

    def attach(self, slot: int, row: np.ndarray):
        """Map a detached row into `slot`, which runs no request: the pages it still maps (a retired prefix) are
        released first, and the slot becomes live."""
        self._undetach(row)
        self.retired.pop(slot, None)
        self.release(slot)
        self.on_reclaim(slot)
        self.table[slot] = row
        self.dirty = True

    def drop(self, row: np.ndarray):
        """Give up a detached row: its references are released, pages nobody else maps return to the free list."""
        self._undetach(row)
        pages = row[row >= 0]
        self.ref[pages] -= 1
        self.free.extend(pages[self.ref[pages] == 0].tolist())

    def hold(self, slot: int, end: int, start: int = 0):
        """Make `slot` live without mapping anything yet, and release its pages past position `end` as well as the
        pages from `start` on that other slots map too (they would be replaced by pages of their own, nothing kept)."""
        self.retired.pop(slot, None)
        n = kv_pages_for(max(int(end), 0))
        self._unmap(slot, n)
        row = self.table[slot]
        for j in range(kv_pages_for(max(int(start), 0)), n):
            p = int(row[j])
            if p >= 0 and self.ref[p] > 1:
                row[j] = -1
                self.ref[p] -= 1
                self.dirty = True

    def share(self, dst: int, src, n_pages: int):
        """Map the first `n_pages` pages of `src` into `dst` as well (a shared prompt prefix). `src`: a slot, or a
        row outside the table (CachedRow.row)."""
        src_row = src if isinstance(src, np.ndarray) else self.table[src]
        for j in range(n_pages):
            p = int(src_row[j])
            if p < 0 or p == self.table[dst, j]:
                continue
            old = int(self.table[dst, j])
            if old >= 0:
                self.ref[old] -= 1
                if self.ref[old] == 0:
                    self.free.append(old)
            self.table[dst, j] = p
            self.ref[p] += 1
            self.dirty = True

    def _take(self) -> int:
        p = self.free.pop()
        self.ref[p] = 1
        self.dirty = True
        return p

    def reserve(self, slot: int, end: int, start: int = 0):
        """Make `slot` live with private pages for every position in [start, end) it is about to write, and mapped
        pages for [0, start). A page overlapping [start, end) that other slots map too is replaced by a private copy of
        its positions before `start` (copy-on-write). Pages past `end` are released."""
        end = max(int(end), 0)
        start = min(max(int(start), 0), end)
        n = kv_pages_for(end)
        if n > self.pages_per_slot:
            raise ValueError(f"{end} positions exceed the slot's KV capacity ({self.pages_per_slot * KV_PAGE})")
        self.hold(slot, end, start)
        row = self.table[slot]
        first = start // KV_PAGE
        while True:
            head = row[first:n]
            cow = (first + np.nonzero((head >= 0) & (self.ref[np.maximum(head, 0)] > 1))[0]).tolist()
            missing = np.nonzero(row[:n] < 0)[0].tolist()
            need = len(cow) + len(missing)
            if len(self.free) >= need:
                break
            if self.retired:
                victim = next(iter(self.retired))
                del self.retired[victim]
                self.release(victim)
                self.on_reclaim(victim)
            elif self.cached:
                # least recently used first; a donor of the admission being reserved only when nothing else is left
                self.drop_cached(next((e for e in self.cached if e not in self.held), next(iter(self.cached))))
                self.evictions += 1
            else:
                raise RuntimeError(
                    f"KV page pool exhausted: slot {slot} needs {need} more pages of {KV_PAGE} positions for {end} "
                    f"positions, {len(self.free)} of the pool's {self.n_pages} pages (kv_pages) are free")
        for j in cow:
            old, new = int(row[j]), self._take()
            keep = min(max(0, start - j * KV_PAGE), KV_PAGE)
            if keep:
                self.copy_page(old, new, keep)
            self.ref[old] -= 1  # another slot still maps it
            row[j] = new
        for j in missing:
            row[j] = self._take()
        self.peak = max(self.peak, self.in_use())

    # ---- prefix cache: prompt prefixes kept after their slot moved on ---------------------------------------------
    def touch(self, entry: CachedRow):
        """`entry` was just inserted or reused: it becomes the most recently used."""
        self.tick += 1
        entry.stamp = self.tick
        self.cached.pop(entry, None)
        self.cached[entry] = None

    def insert(self, slot: int, tokens: torch.Tensor):
        """The retiring `slot` holds the K/V its prefill wrote for `tokens` [C+1, n] at positions [0, n): keep the
        pages of those positions as a cached row, then release the slot's row, so that pages only its decode frames
        wrote go back to the free list. A cached row that already covers the prefix is only touched; cached rows that
        are a prefix of it are dropped. A prefix shorter than one hash block is not kept."""
        rows = np.ascontiguousarray(tokens.numpy().T, dtype=np.int32)
        n = rows.shape[0]
        keys = _chain_keys(rows)
        if keys and (self.table[slot, :kv_pages_for(n)] >= 0).all():
            cover = next((e for e in self._index.get(keys[-1], ()) if e.n >= n and _common_rows(rows, e.rows) >= n),
                         None)
            if cover is not None:
                self.touch(cover)
            else:
                for j, k in enumerate(keys):
                    for e in list(self._index.get(k, ())):
                        if len(e.keys) == j + 1 and e.n <= n and _common_rows(rows, e.rows) >= e.n:
                            self.drop_cached(e)
                row = np.full(self.pages_per_slot, -1, dtype=np.int32)
                m = kv_pages_for(n)
                row[:m] = self.table[slot, :m]
                self.ref[row[:m]] += 1
                entry = CachedRow(row, rows, n, keys)
                for k in keys:
                    self._index.setdefault(k, set()).add(entry)
                self.touch(entry)
        self.release(slot)

    def lookup(self, rows: np.ndarray) -> tuple[int, Optional[CachedRow]]:
        """(rows, cached row) of the longest prefix of token rows [T, C+1] that a cached row holds; (0, None) below
        one hash block. The chain keys narrow the search to the cached rows that share the prompt's deepest matching
        block; an exact compare confirms the one chosen."""
        cands, depth = (), 0
        for j, k in enumerate(_chain_keys(rows)):
            c = self._index.get(k)
            if not c:
                break
            cands, depth = c, j + 1
        lo = depth * PREFIX_BLOCK
        best, hit = 0, None
        for e in cands:  # all of them share rows [0, lo) with the prompt; each diverges within the next block
            n = lo + _common_rows(rows[lo:lo + PREFIX_BLOCK], e.rows[lo:lo + PREFIX_BLOCK])
            if n > best:
                best, hit = n, e
        if hit is not None and _common_rows(rows[:lo], hit.rows[:lo]) < lo:  # a hash collision: compare everything
            best, hit = 0, None
            for e in self.cached:
                n = _common_rows(rows, e.rows)
                if n > best:
                    best, hit = n, e
        return best, hit

    def drop_cached(self, entry: CachedRow):
        """Forget a cached row: pages no slot, parked row or other cached row maps return to the free list."""
        del self.cached[entry]
        self.held.discard(entry)
        for k in entry.keys:
            s = self._index[k]
            s.discard(entry)
            if not s:
                del self._index[k]
        pages = entry.row[entry.row >= 0]
        self.ref[pages] -= 1
        self.free.extend(pages[self.ref[pages] == 0].tolist())

    def drop_cache(self):
        for e in list(self.cached):
            self.drop_cached(e)

    def cached_pages(self) -> int:
        """Pages at least one cached row maps."""
        if not self.cached:
            return 0
        pages = np.concatenate([e.row for e in self.cached])
        return len(np.unique(pages[pages >= 0]))


@dataclass(eq=False)
class ParkedSlot:
    """A request taken out of its slot between two frames (LmEngine.park_slot): everything it needs to continue in
    any slot of the same engine. Its K/V stays in the pool pages `row` references; nothing was copied."""

    blob: torch.Tensor  # device bytes written by fsb_lm_slot_save
    row: np.ndarray  # its detached page-table row (KvPagePool.detach)
    tokens: Optional[torch.Tensor]  # prompt rows whose K/V the pages hold, for prefix reuse once it has a slot again
    covered: Optional[int]  # pages its reservation mapped
    ctx_len: int  # upper bound of its context length, kept for the scheduler


class LmEngine:
    """One model replica on one GPU: weights (bf16, device), KV caches and workspaces (library-owned)."""

    def __init__(self, config, state_dict: dict, device, im_end_id: int, max_batch: int = 1,
                 kv_len: Optional[int] = None, max_rows: int = 2048, max_frames: Optional[int] = None,
                 debug: bool = False, kv_pages: Optional[int] = None, attn_split: int = 0, prefix_cache: bool = False):
        """`kv_len`: KV positions one sequence can hold. `kv_pages`: size of the slow KV cache's page pool (pages of
        64 positions); None = room for every slot at full capacity, so that no reservation can fail. `attn_split`:
        0 = off; else a multiple of 64: a decode row with a longer context has its attention split into spans of that
        many positions over several CTAs (include/fishb200.h fsb_lm_config.attn_split). `prefix_cache`: the prompt
        pages of a request that `prefill_reusing` admitted stay in the pool after its slot moves on, as a prefix later
        requests reuse until the pool needs the pages (KvPagePool.insert); off: a prefix lives as long as its slot
        holds it."""
        if not torch.cuda.is_available():
            raise _lib.FsbError("fish_speech_b200 needs a CUDA device (sm_90a); there is no CPU path")
        self.lib = _lib.lib()
        self.cfg = config
        self.im_end_id = int(im_end_id)
        self.device = torch.device(device)
        kv_len = int(kv_len or config.max_seq_len)
        kv_len = min(kv_len, config.max_seq_len)
        max_frames = int(max_frames or kv_len)
        self.max_batch, self.kv_len, self.max_rows, self.max_frames = max_batch, kv_len, max_rows, max_frames
        self.row_tile = decode_row_tile(max_batch)
        self._keep = []  # device tensors the library points into
        dev = self.device

        def put(t: torch.Tensor) -> int:
            t = t.detach().to(device=dev, dtype=torch.bfloat16).contiguous()
            self._keep.append(t)
            return t.data_ptr()

        sd = state_dict
        c = config

        def layer_struct(prefix: str) -> _lib.LmLayer:
            L = _lib.LmLayer()
            L.d_attn_norm = put(sd[f"{prefix}.attention_norm.weight"])
            L.d_wqkv = put(sd[f"{prefix}.attention.wqkv.weight"])
            L.d_bqkv = put(sd[f"{prefix}.attention.wqkv.bias"]) if f"{prefix}.attention.wqkv.bias" in sd else None
            L.d_q_norm = put(sd[f"{prefix}.attention.q_norm.weight"]) if f"{prefix}.attention.q_norm.weight" in sd else None
            L.d_k_norm = put(sd[f"{prefix}.attention.k_norm.weight"]) if f"{prefix}.attention.k_norm.weight" in sd else None
            L.d_wo = put(sd[f"{prefix}.attention.wo.weight"])
            L.d_bo = put(sd[f"{prefix}.attention.wo.bias"]) if f"{prefix}.attention.wo.bias" in sd else None
            L.d_ffn_norm = put(sd[f"{prefix}.ffn_norm.weight"])
            # fused gate|up projection, rows interleaved so that SwiGLU runs in the GEMM epilogue
            L.d_w13 = put(interleave_w13(sd[f"{prefix}.feed_forward.w1.weight"], sd[f"{prefix}.feed_forward.w3.weight"]))
            L.d_w2 = put(sd[f"{prefix}.feed_forward.w2.weight"])
            return L

        self._layers = (_lib.LmLayer * c.n_layer)(*[layer_struct(f"layers.{i}") for i in range(c.n_layer)])
        self._fast_layers = (_lib.LmLayer * c.n_fast_layer)(
            *[layer_struct(f"fast_layers.{i}") for i in range(c.n_fast_layer)])
        head_src = sd["embeddings.weight"] if c.tie_word_embeddings else sd["output.weight"]
        # Only the semantic ids and <|im_end|> survive the reference's -inf logit bias
        # (inference.py:308-320): the head is restricted to those rows.
        head = torch.cat([head_src[c.semantic_begin_id: c.semantic_end_id + 1],
                          head_src[self.im_end_id: self.im_end_id + 1]], 0)
        W = _lib.LmWeights()
        W.d_embeddings = put(sd["embeddings.weight"])
        W.d_codebook_embeddings = put(sd["codebook_embeddings.weight"])
        W.d_norm = put(sd["norm.weight"])
        W.d_head = put(head)
        W.head_rows = head.shape[0]
        W.d_freqs = put(rope_table(kv_len, c.head_dim, c.rope_base))
        W.layers = self._layers
        W.d_fast_embeddings = put(sd["fast_embeddings.weight"])
        W.d_fast_norm = put(sd["fast_norm.weight"])
        W.d_fast_output = put(sd["fast_output.weight"])
        W.d_fast_freqs = put(rope_table(c.num_codebooks, c.fast_head_dim, c.rope_base))
        if "fast_project_in.weight" in sd:
            W.d_fast_proj_w = put(sd["fast_project_in.weight"])
            W.d_fast_proj_b = put(sd["fast_project_in.bias"])
        W.fast_layers = self._fast_layers
        self.head_rows = head.shape[0]

        K = _lib.LmConfig()
        K.dim, K.n_layer, K.n_head, K.n_kv_head, K.head_dim, K.intermediate = (
            c.dim, c.n_layer, c.n_head, c.n_local_heads, c.head_dim, c.intermediate_size)
        (K.fast_dim, K.n_fast_layer, K.fast_n_head, K.fast_n_kv_head, K.fast_head_dim, K.fast_intermediate) = (
            c.fast_dim, c.n_fast_layer, c.fast_n_head, c.fast_n_local_heads, c.fast_head_dim, c.fast_intermediate_size)
        K.vocab_size, K.codebook_size, K.num_codebooks = c.vocab_size, c.codebook_size, c.num_codebooks
        K.semantic_begin_id, K.semantic_end_id, K.im_end_id = c.semantic_begin_id, c.semantic_end_id, self.im_end_id
        K.norm_eps = c.norm_eps
        K.qk_norm, K.fast_qk_norm = int(c.attention_qk_norm), int(c.fast_attention_qk_norm)
        K.scale_codebook_embeddings = int(c.scale_codebook_embeddings)
        K.norm_fastlayer_input = int(getattr(c, "norm_fastlayer_input", False))
        K.max_batch, K.kv_len, K.max_rows, K.max_frames, K.debug = max_batch, kv_len, max_rows, max_frames, int(debug)
        pages_per_slot = kv_pages_for(kv_len)
        K.kv_pages = int(kv_pages) if kv_pages else max_batch * pages_per_slot
        K.attn_split = self.attn_split = int(attn_split or 0)
        self._K, self._W = K, W
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.fsb_lm_create(C.byref(K), C.byref(W), C.byref(h)))
        self.h = h
        self.debug = debug
        self._views = {}
        self._ctx_bound = 0  # upper bound of every slot's length, tracked on the host
        self.slot_control = False
        self._slot_tokens: dict = {}  # slot -> token rows [C+1, T] (CPU int32) whose K/V positions [0, T) are valid
        self.rows_reused = 0
        self.rows_prefilled = 0
        self.kv_pool = KvPagePool(max_batch, pages_per_slot, K.kv_pages, copy_page=self._copy_page,
                                  on_reclaim=self._forget_slot, prefix_cache=prefix_cache)
        self._wfrom: dict = {}  # slot -> lowest position the next decode frames write (copy-on-write bound)
        self._covered: dict = {}  # slot -> pages [0, n) its last reservation mapped (decode skips what is covered)

    def close(self):
        if getattr(self, "h", None):
            self.lib.fsb_lm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- decode row tile (include/fishb200.h fsb_lm_set_decode_tile) -------------------------------------------------
    def set_decode_tile(self, tile: int) -> None:
        """Test hook: 0 = each frame runs the 32-row step GEMMs when it decodes <= 32 rows (the default), 32 or 64 =
        that tile for every frame. The tiles give the same bits; only the frame time differs."""
        _lib.check(self.lib.fsb_lm_set_decode_tile(self.h, int(tile)))

    @property
    def decode_tile(self) -> int:
        """Row tile of the last `decode` call (0 before the first)."""
        return int(self.lib.fsb_lm_decode_tile(self.h))

    @property
    def graph_captures(self) -> int:
        """Decode frames captured into CUDA graphs since the engine was created."""
        return int(self.lib.fsb_lm_graph_captures(self.h))

    # -------------------------------------------------------------------------------------------
    def buffer(self, name: str) -> torch.Tensor:
        """Zero-copy torch view of a named device buffer of the handle."""
        if name in self._views:
            return self._views[name]
        ptr, nbytes = C.c_void_p(), C.c_size_t()
        _lib.check(self.lib.fsb_lm_buffer(self.h, name.encode(), C.byref(ptr), C.byref(nbytes)))
        c = self.cfg
        C1 = c.num_codebooks + 1
        rt = self.row_tile
        R = max(self.max_rows, 128)
        shapes = {
            "out_tokens": ((self.max_batch, C1, self.max_frames), "<i4"),
            "n_out": ((self.max_batch,), "<i4"),
            "pos": ((self.row_tile,), "<i4"),
            "step": ((1,), "<i8"),
            "finished": ((self.max_batch,), "<i4"),
            "cur_tok": ((self.max_batch, C1), "<i4"),
            "ras_window": ((self.max_batch, 10), "<i4"),
            "slot_state": ((self.max_batch,), "<i4"),
            "slot_limit": ((self.max_batch,), "<i4"),
            "slot_temperature": ((self.max_batch,), "<f4"),
            "slot_top_p": ((self.max_batch,), "<f4"),
            "slot_top_k": ((self.max_batch,), "<i4"),
            "slot_seed": ((self.max_batch,), "<i8"),
            "kv_miss": ((self.max_batch,), "<i4"),
            "kv_page": ((self.max_batch, self.kv_pool.pages_per_slot), "<i4"),
            "slow_logits": ((self.max_batch, self.head_rows), "<f4"),
            "fast_logits": ((c.num_codebooks, self.max_batch, c.codebook_size), "<f4"),
            # decode state (include/fishb200.h fsb_lm_test_layer_gemms), row_tile rows; "attn" / "ffn_h" are flat:
            # the rows of the stack being run sit at stride H*Dh / I of that stack
            "x_slow": ((rt, c.dim), "<u2"),
            "x_fast": ((rt, c.fast_dim), "<u2"),
            "ssq_slow": ((rt, 32), "<f4"),
            "ssq_fast": ((rt, 32), "<f4"),
            "attn": ((rt * max(c.n_head * c.head_dim, c.fast_n_head * c.fast_head_dim),), "<u2"),
            "q": ((rt * max(c.n_head * c.head_dim, c.fast_n_head * c.fast_head_dim),), "<u2"),
            # split attention: one record per (slot, KV head, span of the launch); the span count follows the bound
            "attn_span_ws": ((nbytes.value // 4,), "<f4"),
            "ffn_h": ((rt * max(c.intermediate_size, c.fast_intermediate_size),), "<u2"),
            # KV caches (include/fishb200.h fsb_lm_test_layer_attn): the slow page pool, the fast stack per slot
            "k_slow": ((c.n_layer, self._K.kv_pages, c.n_local_heads, KV_PAGE, c.head_dim), "<u2"),
            "v_slow": ((c.n_layer, self._K.kv_pages, c.n_local_heads, KV_PAGE, c.head_dim), "<u2"),
            "k_fast": ((c.n_fast_layer, self.max_batch, c.fast_n_local_heads, c.num_codebooks, c.fast_head_dim), "<u2"),
            "v_fast": ((c.n_fast_layer, self.max_batch, c.fast_n_local_heads, c.num_codebooks, c.fast_head_dim), "<u2"),
            # prefill workspaces (include/fishb200.h fsb_lm_test_prefill_stage), R = max(max_rows, 128) token rows;
            # "ws_prefill" is flat: the last prefill GEMM's fp32 result [rows][n_out] at row stride n_out
            "x_prefill": ((R, c.dim), "<u2"),
            "xn_prefill": ((R, c.dim), "<u2"),
            "q_prefill": ((R, c.n_head, c.head_dim), "<u2"),
            "attn_prefill": ((R, c.n_head * c.head_dim), "<u2"),
            "h_prefill": ((R, c.intermediate_size), "<u2"),
            "ws_prefill": ((nbytes.value // 4,), "<f4"),
            # frame tail (include/fishb200.h fsb_lm_test_frame_stage): the fast_project_in operand, rows at stride dim;
            # fused admission's staged last prompt rows, by slot
            "fast_hidden": ((rt * max(c.dim, c.fast_dim),), "<u2"),
            "first_frame_x": ((self.max_batch, c.dim), "<u2"),
            "first_frame_ssq": ((self.max_batch, 32), "<f4"),
            "first_frame_pos": ((self.max_batch,), "<i4"),
            "first_frame_pending": ((self.max_batch,), "<i4"),
        }
        shape, ts = shapes[name]
        with torch.cuda.device(self.device):
            t = torch.as_tensor(_DevView(ptr.value, shape, ts), device=self.device)
        if ts == "<u2":
            t = t.view(torch.bfloat16)
        self._views[name] = t
        return t

    def sampling(self, temperature: float, top_p: float, top_k: int, seed: int = 0) -> _lib.Sampling:
        s = _lib.Sampling()
        s.temperature = bf16_round(temperature)
        s.top_p = bf16_round(top_p)
        s.top_k = int(top_k)
        s.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        return s

    def _grow_bound(self, n: int):
        n = min(int(n), self.kv_len)
        if n > self._ctx_bound:
            self._ctx_bound = n
        _lib.check(self.lib.fsb_lm_set_context_bound(self.h, self._ctx_bound))

    def set_context_bound(self, n: int):
        """For callers that place tokens at explicit positions (decode_one_token_ar / decode_n_tokens)."""
        self._grow_bound(n)

    def set_context_bound_exact(self, n: int):
        """For a scheduler that knows every live slot's length: the bound may also shrink."""
        self._ctx_bound = 0
        self._grow_bound(max(1, n))

    def set_slot_control(self, enable: bool):
        """Per-slot sampling parameters / stop rule / RNG stream (include/fishb200.h fsb_lm_set_slot_control)."""
        _lib.check(self.lib.fsb_lm_set_slot_control(self.h, int(bool(enable))))
        self.slot_control = bool(enable)

    def set_sampler_noise(self, u: Optional[torch.Tensor]):
        """Test hook (include/fishb200.h fsb_lm_set_sampler_noise): u fp32 [frames][draws][ld] on the device."""
        if u is None:
            self._noise = None
            _lib.check(self.lib.fsb_lm_set_sampler_noise(self.h, None, 0, 0))
            return
        u = u.to(device=self.device, dtype=torch.float32).contiguous()
        self._noise = u
        _lib.check(self.lib.fsb_lm_set_sampler_noise(self.h, u.data_ptr(), u.shape[1], u.shape[2]))

    def test_sample(self, logits: torch.Tensor, sp: Optional[_lib.Sampling], codebook: int = 0,
                    row_slot: Optional[torch.Tensor] = None, use_ras: bool = False):
        """Test hook (include/fishb200.h fsb_lm_test_sample): the sampler alone on fp32 logits [rows][n], behind the
        slow head (codebook 0) or fast codebook `codebook`; row_slot int32 [rows] on the device or None."""
        logits = logits.to(device=self.device, dtype=torch.float32).contiguous()
        rs = None if row_slot is None else row_slot.to(device=self.device, dtype=torch.int32).contiguous()
        _lib.check(self.lib.fsb_lm_test_sample(self.h, int(codebook > 0), int(codebook), logits.shape[0],
                                               None if rs is None else rs.data_ptr(), logits.data_ptr(),
                                               int(bool(use_ras)), None if sp is None else C.byref(sp), _stream()))

    PREFILL_STAGES = ("embed", "qkv", "attn", "wo", "w13", "w2")

    def test_prefill_stage(self, stage: str, rows: int, layer: int = 0, tokens: Optional[torch.Tensor] = None,
                           row_seq: Optional[torch.Tensor] = None, row_pos: Optional[torch.Tensor] = None):
        """Test hook (include/fishb200.h fsb_lm_test_prefill_stage): one stage of slow layer `layer` of the prefill
        over `rows` token rows, on the prefill buffers as they are. tokens int32 [rows][C+1] (embed); row_seq / row_pos
        int32 [rows] (qkv, attn). Returns after the stage has finished."""
        def dev(t):
            return None if t is None else t.to(device=self.device, dtype=torch.int32).contiguous()

        tok, seq, pos = dev(tokens), dev(row_seq), dev(row_pos)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.fsb_lm_test_prefill_stage(
                self.h, int(layer), self.PREFILL_STAGES.index(stage), int(rows), *(
                    None if t is None else t.data_ptr() for t in (tok, seq, pos)), _stream()))
            torch.cuda.current_stream().synchronize()

    FRAME_STAGES = ("embed", "splice", "head", "fast_in", "fast_embed", "fast_head", "end")

    def test_frame_stage(self, stage: str, rows: int, tile: Optional[int] = None, p: int = 0,
                         row_slot: Optional[torch.Tensor] = None, set_pos_rows: Optional[torch.Tensor] = None,
                         row_pos_src: Optional[torch.Tensor] = None, first_frame: bool = False,
                         sp: Optional[_lib.Sampling] = None):
        """Test hook (include/fishb200.h fsb_lm_test_frame_stage): one launch group of a decode frame around its stacks
        over `rows` rows on the plans of row tile `tile` (default: the engine's), on the buffers as they are; fast pass
        `p` for fast_embed / fast_head. row_slot / set_pos_rows / row_pos_src int32 on the device or None. Returns after
        the stage has finished."""
        def dev(t):
            return None if t is None else t.to(device=self.device, dtype=torch.int32).contiguous()

        rs, spr, rps = dev(row_slot), dev(set_pos_rows), dev(row_pos_src)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.fsb_lm_test_frame_stage(
                self.h, self.FRAME_STAGES.index(stage), int(tile or self.row_tile), int(rows), int(p),
                *(None if t is None else t.data_ptr() for t in (rs, spr, rps)), int(bool(first_frame)),
                None if sp is None else C.byref(sp), _stream()))
            torch.cuda.current_stream().synchronize()

    # ---- paged slow KV cache (KvPagePool) --------------------------------------------------------------------------
    def _forget_slot(self, slot: int):
        """The pool reclaimed the slot's pages: its prefix record and reservation are gone."""
        self._slot_tokens.pop(slot, None)
        self._covered.pop(slot, None)

    def _copy_page(self, src: int, dst: int, n: int):
        _lib.check(self.lib.fsb_lm_copy_kv_page(self.h, src, dst, n, _stream()))

    def _reserve(self, items):
        """items: (slot, end, start) -- map pages for positions [0, end) of each slot, private from `start` on. Every
        slot is first made live and trimmed to its end, so that none of them is reclaimed for another; the page table
        then reaches the device with one stream-ordered copy."""
        pool = self.kv_pool
        with torch.cuda.device(self.device):
            for s, end, start in items:
                pool.hold(int(s), end, start)
            for s, end, start in items:
                pool.reserve(int(s), end, start)
                self._covered[int(s)] = kv_pages_for(end)
            if pool.dirty:
                table = torch.from_numpy(pool.table.copy()).pin_memory()
                self.buffer("kv_page").copy_(table, non_blocking=True)
                pool.dirty = False

    def reserve(self, slot: int, n_positions: int, start: int = 0):
        """Pages for every position < n_positions of `slot`, before it writes [start, n_positions): for callers that
        decode at explicit positions (decode_one_token_ar / decode_n_tokens)."""
        n_positions = min(int(n_positions), self.kv_len)
        self._reserve([(slot, n_positions, start)])
        self._wfrom[int(slot)] = int(start)

    def grow_kv(self, ends: dict):
        """ends: {slot: end} -- map pages for positions [covered end, end) of each live slot, which has written nothing
        past what its pages cover; one page-table upload for all of them. Only retired rows are reclaimed."""
        self._reserve([(int(s), int(e), self._covered.get(int(s), 0) * KV_PAGE) for s, e in ends.items()
                       if kv_pages_for(e) > self._covered.get(int(s), 0)])

    def retire_slot(self, slot: int, cache: bool = True):
        """The slot's request is done: its pages stay mapped as a reusable prefix until the pool needs them. With the
        prefix cache, a slot that holds a prompt record (prefill_reusing) moves the pages of that prompt into the cache
        instead and gives the rest back; `cache=False` (a request whose tokens are void) keeps it out of the cache."""
        slot = int(slot)
        tokens = self._slot_tokens.get(slot)
        if cache and tokens is not None and self.kv_pool.prefix_cache:
            self.kv_pool.insert(slot, tokens)
            self._forget_slot(slot)
        self.kv_pool.retire(slot)

    @property
    def prefix_cache(self) -> bool:
        return self.kv_pool.prefix_cache

    @property
    def prefix_hits(self) -> int:
        """Admissions that mapped a prefix from the prefix cache."""
        return self.kv_pool.hits

    @property
    def prefix_evictions(self) -> int:
        """Cached prefixes dropped because a reservation needed their pages."""
        return self.kv_pool.evictions

    @property
    def pages_cached(self) -> int:
        """Pool pages the prefix cache maps now."""
        return self.kv_pool.cached_pages()

    def park_slot(self, slot: int, ctx_len: int = 0) -> ParkedSlot:
        """Take the request running in `slot` out of it, between two frames: its per-slot decode state goes into a
        device blob (one small kernel, which also idles the row), its page-table row is detached with its pages, and
        the slot is free for another request. `resume_slot` continues it in any slot with the same bits."""
        slot = int(slot)
        with torch.cuda.device(self.device):
            blob = torch.empty(int(self.lib.fsb_lm_slot_blob_bytes(self.h)), dtype=torch.uint8, device=self.device)
            _lib.check(self.lib.fsb_lm_slot_save(self.h, slot, blob.data_ptr(), _stream()))
        parked = ParkedSlot(blob, self.kv_pool.detach(slot), self._slot_tokens.pop(slot, None),
                            self._covered.pop(slot, None), int(ctx_len))
        self._reserve([])  # the emptied row reaches the device before the slot's next request
        return parked

    def resume_slot(self, slot: int, parked: ParkedSlot):
        """Continue a parked request in `slot` (idle; what it still maps as a retired prefix is released)."""
        slot = int(slot)
        self.kv_pool.attach(slot, parked.row)
        if parked.tokens is not None:
            self._slot_tokens[slot] = parked.tokens
        if parked.covered is not None:
            self._covered[slot] = parked.covered
        self._reserve([])
        with torch.cuda.device(self.device):
            _lib.check(self.lib.fsb_lm_slot_restore(self.h, slot, parked.blob.data_ptr(), _stream()))

    def drop_parked(self, parked: ParkedSlot):
        """A parked request will not continue: its pages go back to the pool."""
        self.kv_pool.drop(parked.row)

    def release_kv(self):
        """Forget every slot's K/V and the prefix cache: all pages return to the pool."""
        self._slot_tokens.clear()
        self._covered.clear()
        self.kv_pool.drop_cache()
        for s in range(self.max_batch):
            self.kv_pool.release(s)
            self.kv_pool.retire(s)
        self._reserve([])

    def _donor(self, prompt: torch.Tensor, slot: int, busy) -> tuple[int, object]:
        """(rows, donor) of the longest prefix of `prompt` whose K/V a slot holds -- its own, or one not in `busy` --
        or the prefix cache does: the donor is a slot or a CachedRow."""
        best, donor = 0, slot
        for d, toks in self._slot_tokens.items():
            if d != slot and d in busy:
                continue
            n = self._common_prefix(prompt, toks)
            if n > best:
                best, donor = n, d
        if self.kv_pool.cached:
            n, entry = self.kv_pool.lookup(np.ascontiguousarray(prompt.numpy().T, dtype=np.int32))
            if n > best:
                best, donor = n, entry
        best = min(best, prompt.shape[1] - 1)  # at least the last row is computed: its logits are sampled
        return (best, donor) if best >= self.MIN_REUSE else (0, slot)

    def kv_pages_needed(self, prompt: torch.Tensor, n_positions: int, slot: int, busy=(), reuse: bool = False) -> int:
        """Pages a request in `slot` adds to those live slots map: all of [0, n_positions), less the whole pages of a
        prefix it shares with a live slot (prefill_reusing). A prefix from a retired slot or the prefix cache is not
        subtracted: its pages count as available, and sharing them makes them live. `prompt`: the request's token rows
        on the host."""
        need = kv_pages_for(min(int(n_positions), self.kv_len))
        if reuse:
            best, donor = self._donor(prompt, int(slot), set(busy) | {int(slot)})
            if isinstance(donor, int) and donor != slot and donor not in self.kv_pool.retired:
                need -= best // KV_PAGE
        return need

    def kv_pages_available(self) -> int:
        return self.kv_pool.available()

    def reset(self):
        for s in range(self.max_batch):
            self.retire_slot(s)  # their K/V stays mapped (or cached) for prefix reuse until the pool needs the pages
        self._ctx_bound = 0
        with torch.cuda.device(self.device):
            _lib.check(self.lib.fsb_lm_reset(self.h, _stream()))

    def prefill(self, prompts: Sequence[torch.Tensor], slots: Sequence[int], sp: Optional[_lib.Sampling],
                start_pos: Optional[Sequence[int]] = None, do_sample: bool = True,
                kv_end: Optional[Sequence[int]] = None, defer_first_frame: bool = False) -> None:
        """prompts[k]: integer tensor [C+1, T_k] (row 0 token ids, rows 1..C codes) for slot slots[k]. `kv_end[k]`:
        reserve KV pages up to that position (prompt + frames to come) instead of the prompt alone.
        `defer_first_frame` (with do_sample, under slot control): the first frames are not run here; the next `decode`
        runs them as rows of its first frame, next to the running requests, with the same tokens
        (include/fishb200.h fsb_lm_prefill_deferred)."""
        if defer_first_frame and not self.slot_control:
            raise ValueError("defer_first_frame needs slot control (set_slot_control)")
        C1 = self.cfg.num_codebooks + 1
        start_pos = list(start_pos) if start_pos is not None else [0] * len(prompts)
        for p, s0 in zip(prompts, start_pos):
            if p.shape[0] != C1:
                raise ValueError(f"prompt must have {C1} rows, got {tuple(p.shape)}")
            if s0 + p.shape[1] > self.kv_len:
                raise ValueError(f"Input sequence length {s0 + p.shape[1]} exceeds the KV cache ({self.kv_len})")
        # group whole sequences into passes of <= max_rows rows; a longer sequence is split in time
        groups, cur, cur_rows = [], [], 0
        for k, p in enumerate(prompts):
            T = p.shape[1]
            t0 = 0
            while T - t0 > self.max_rows:  # time-split: no sampling on non-final pieces
                if cur:
                    groups.append(cur)
                    cur, cur_rows = [], 0
                groups.append([(k, t0, t0 + self.max_rows, False)])
                t0 += self.max_rows
            if cur_rows + (T - t0) > self.max_rows:
                groups.append(cur)
                cur, cur_rows = [], 0
            cur.append((k, t0, T, True))
            cur_rows += T - t0
        if cur:
            groups.append(cur)
        dev = self.device
        for k, s0 in enumerate(start_pos):
            if s0 == 0:
                self._slot_tokens.pop(int(slots[k]), None)  # overwritten from position 0: the old record is void
        ends = [s0 + p.shape[1] for p, s0 in zip(prompts, start_pos)]
        if kv_end is not None:
            ends = [max(e, min(int(k), self.kv_len)) for e, k in zip(ends, kv_end)]
        self._reserve([(int(s), e, s0) for s, e, s0 in zip(slots, ends, start_pos)])
        for p, s, s0 in zip(prompts, slots, start_pos):
            self._wfrom[int(s)] = s0 + p.shape[1]
        self._grow_bound(max(s0 + p.shape[1] for p, s0 in zip(prompts, start_pos)) + 1)
        with torch.cuda.device(dev):
            for grp in groups:
                toks, rslot, rpos, last, gsl = [], [], [], [], []
                rows = 0
                final = all(f for (_, _, _, f) in grp)
                for (k, a, b, _) in grp:
                    p = prompts[k][:, a:b]
                    toks.append(p.t().to(device=dev, dtype=torch.int32))
                    n = b - a
                    rslot.append(torch.full((n,), int(slots[k]), dtype=torch.int32))
                    rpos.append(torch.arange(start_pos[k] + a, start_pos[k] + b, dtype=torch.int32))
                    rows += n
                    last.append(rows - 1)
                    gsl.append(int(slots[k]))
                d_tok = torch.cat(toks).contiguous()
                d_slot = torch.cat(rslot).to(dev)
                d_pos = torch.cat(rpos).to(dev)
                d_last = torch.tensor(last, dtype=torch.int32, device=dev)
                d_gsl = torch.tensor(gsl, dtype=torch.int32, device=dev)
                if defer_first_frame and do_sample and final:
                    h_gsl = (C.c_int32 * len(gsl))(*gsl)
                    _lib.check(self.lib.fsb_lm_prefill_deferred(
                        self.h, d_tok.data_ptr(), d_slot.data_ptr(), d_pos.data_ptr(), rows, d_last.data_ptr(),
                        d_gsl.data_ptr(), len(grp), h_gsl, _stream()))
                else:
                    _lib.check(self.lib.fsb_lm_prefill(
                        self.h, d_tok.data_ptr(), d_slot.data_ptr(), d_pos.data_ptr(), rows, d_last.data_ptr(),
                        d_gsl.data_ptr(), len(grp), int(do_sample and final), C.byref(sp) if sp is not None else None,
                        _stream()))
                # index tensors must outlive the asynchronous kernels that read them
                self._inflight = (d_tok, d_slot, d_pos, d_last, d_gsl)

    # ---- prefix KV reuse (include/fishb200.h fsb_lm_copy_kv; SURVEY §8(f).2) -----------------------------------
    MIN_REUSE = 16  # shorter shared prefixes are not worth a separate prefill pass

    @staticmethod
    def _common_prefix(a: torch.Tensor, b: torch.Tensor) -> int:
        n = min(a.shape[1], b.shape[1])
        if n == 0:
            return 0
        diff = (a[:, :n] != b[:, :n]).any(dim=0).nonzero()
        return int(diff[0]) if len(diff) else n

    def prefill_reusing(self, prompts: Sequence[torch.Tensor], slots: Sequence[int], sp: Optional[_lib.Sampling],
                        do_sample: bool = True, kv_end: Optional[Sequence[int]] = None,
                        defer_first_frame: bool = False) -> list[int]:
        """`prefill` of full prompts that skips every row whose K/V the cache already holds: the longest prefix
        a prompt shares with what its own slot was last prefilled with, or with another slot that is not being
        re-prefilled in this call (its whole pages are mapped by reference; a partly shared last page is copied).
        The reference re-prefills the whole growing conversation for every chunk of `generate_long`
        (inference.py:611-721); prefill is row-independent, so the reused K/V is bit-identical to what a full
        prefill would write. `defer_first_frame` as for `prefill`. Returns the reused length per prompt."""
        host = [p.detach().to("cpu", torch.int32) for p in prompts]
        busy = set(int(s) for s in slots)
        ends = [p.shape[1] if kv_end is None else max(p.shape[1], min(int(e), self.kv_len))
                for p, e in zip(host, kv_end if kv_end is not None else host)]
        for s, e in zip(slots, ends):
            self.kv_pool.hold(int(s), e, e)  # no slot of this call is reclaimed for another
        reused, pieces = [], []
        pool = self.kv_pool
        for p, s in zip(host, slots):  # every prefix is mapped before any page is allocated: the pages the slots
            s = int(s)                 # held before (maybe shared among them) are released first
            best, donor = self._donor(p, s, busy)
            if isinstance(donor, CachedRow):
                pool.share(s, donor.row, kv_pages_for(best))
                pool.touch(donor)
                pool.held.add(donor)
                pool.hits += 1
            elif donor != s:
                pool.share(s, donor, kv_pages_for(best))
            reused.append(best)
        try:
            self._reserve([(int(s), e, b) for s, e, b in zip(slots, ends, reused)])
        finally:
            pool.held.clear()
        for p, b in zip(prompts, reused):
            pieces.append(p[:, b:])
        defer = dict(defer_first_frame=True) if defer_first_frame else {}
        self.prefill(pieces, slots, sp, start_pos=reused, do_sample=do_sample, kv_end=ends, **defer)
        for p, s in zip(host, slots):
            self._slot_tokens[int(s)] = p
        self.rows_reused += sum(reused)
        self.rows_prefilled += sum(p.shape[1] - b for p, b in zip(host, reused))
        return reused

    def decode(self, batch: int, nframes: int, sp: Optional[_lib.Sampling], use_graph: bool = True) -> None:
        """Under slot control the scheduler reserved every request's pages at admission; otherwise the frames'
        positions are reserved here, before the call."""
        if not self.slot_control and self._ctx_bound - 1 + nframes > self.kv_len:
            raise ValueError(f"decode: {nframes} more frames from position {self._ctx_bound - 1} run past the KV "
                             f"cache ({self.kv_len} positions)")
        if not self.slot_control:
            end = self._ctx_bound - 1 + nframes
            n = kv_pages_for(min(end, self.kv_len))
            retired = self.kv_pool.retired
            if any(self._covered.get(s, -1) < n or s in retired for s in range(batch)):  # new pages every 64 frames
                self._reserve([(s, end, self._wfrom.get(s, 0)) for s in range(batch)])
        self._grow_bound(self._ctx_bound + nframes)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.fsb_lm_decode(self.h, batch, nframes, C.byref(sp) if sp is not None else None,
                                               int(use_graph), _stream()))
