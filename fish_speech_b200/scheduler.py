"""Continuous batching over the engine's KV slots (SURVEY.md 8f.1).

The reference serves ONE request at a time: `launch_thread_safe_queue` (inference.py:748-799) pops a
request, runs `generate` (prefill, then the `decode_n_tokens` loop with a host-side <|im_end|> test per
frame, inference.py:184-238) to completion, then pops the next one. Here up to `max_slots` requests
share every decode frame: a request is prefilled into a free slot while the others are mid-utterance,
its stop rule runs on the device, and its slot is handed to the next waiting request as soon as it
finishes. The kernels are batch-invariant and a request's random stream depends on its own seed and
frame index only, so every request returns exactly the tokens `generate` would return for it alone.

Paced requests (`SlotRequest.pace`, frames per second the consumer plays) let an engine serve more live streams
than it has slots: a slot produces frames several times faster than they are heard, so a stream that is far
enough ahead of its playback is parked between two polls (its K/V stays in its pool pages, nothing is copied) and
its slot serves a stream that is about to run dry; `schedule_live` is the whole policy.

Compact rows (`ContinuousBatcher(compact_rows=True)`): a frame decodes rows [0, 1 + highest live slot) instead of
every slot, and when the live requests fit in 32 rows the ones above them move down between two polls (the same park /
resume, no K/V copied), so that an engine of more than 32 slots runs its 32-row step GEMMs whenever load allows;
`compact_moves` is the whole policy.

Fused admission (`ContinuousBatcher(fused_admission=True)`): an admitted request is prefilled without its first frame,
which then runs as one more row of the poll's first decode frame (LmEngine.prefill defer_first_frame), with the same
tokens; until that frame has run, the request is neither moved nor parked.
"""
from __future__ import annotations

import threading
import time
from dataclasses import dataclass, field
from typing import Callable, NamedTuple, Optional, Sequence

import torch

from .engine import MAX_DECODE_BATCH, STEP_ROWS, bf16_round, kv_pages_for


class Cancelled(Exception):
    """`SlotRequest.error` of a request taken out by `ContinuousBatcher.cancel`."""


@dataclass
class StreamClock:
    """Playback clock of one utterance, shared by the requests (chunks) that make it up: a later chunk continues the
    clock of the frames already handed out instead of starting as a new arrival."""

    t_first: Optional[float] = None  # when the first frames were handed out
    frames: int = 0  # frames handed out so far


@dataclass(eq=False)  # identity semantics: requests hold tensors
class SlotRequest:
    """One `generate` call waiting for / occupying a slot."""

    prompt: torch.Tensor  # [C+1, T] integer
    max_new_tokens: int
    temperature: float = 1.0
    top_p: float = 0.9
    top_k: int = 30
    seed: int = 0
    reuse_prefix: bool = False  # prefill only the rows whose K/V no slot already holds (LmEngine.prefill_reusing)
    on_done: Optional[Callable[["SlotRequest"], None]] = None
    # streaming (SURVEY 8f.3): called after a poll with the codes [C, k] of frames that are final, in order; over the
    # whole request exactly result[1:, T:-1] (what generate_long keeps, inference.py:708), before on_done
    on_frames: Optional[Callable[["SlotRequest", torch.Tensor], None]] = None
    tag: object = None
    # frames per second the consumer plays; None: FIFO admission, never parked
    pace: Optional[float] = None
    stream: Optional[StreamClock] = None  # one per utterance (made at submit when a paced request has none)
    # filled by the batcher
    result: Optional[torch.Tensor] = None  # [C+1, T+n] like generate()
    error: Optional[BaseException] = None
    done: threading.Event = field(default_factory=threading.Event)
    slot: int = -1
    _limit: int = 0
    _emitted: int = 0
    _host_prompt: Optional[torch.Tensor] = None  # the prompt on the host, for page-limited admission with reuse
    _t_submit: float = 0.0
    _parked: object = None  # engine.ParkedSlot while the request is live without a slot
    parks: int = 0
    resumes: int = 0
    # KV growth (ContinuousBatcher kv_growth): times it waited parked for pages, and its longest such wait (seconds)
    page_parks: int = 0
    page_wait: float = 0.0
    _short_since: float = 0.0
    moves: int = 0  # compact_rows: times it was moved to a lower slot

    def lead(self, now: float) -> float:
        """Frames the consumer holds beyond what it has played at `now` (negative: it is waiting for frames). An
        unpaced request has no playback clock: it is always due."""
        if self.pace is None:
            return float("-inf")
        st = self.stream
        if st is None or st.t_first is None:
            return -self.pace * (now - self._t_submit)
        return st.frames - self.pace * (now - st.t_first)


# Policy thresholds, in polls (multiples of `frames_per_poll` frames of lead). They are choices, not measurements.
# A parked request gets a slot back once less than RESUME_POLLS polls of audio are left with its consumer: after the
# resume its next frames are final one poll later, and a poll of frames takes several times longer to play than to
# make, so one poll of lead is enough not to run dry. A running request may be parked once it is PARK_POLLS polls
# ahead: low enough that a request reaches it well before an utterance of a few seconds ends, or nothing is ever
# parked. The gap of three polls is what keeps requests from flapping: a resumed request gains less than one poll of
# lead per poll (the consumer plays meanwhile), so it runs at least three polls before it can be parked again, and a
# parked one plays three polls' worth of audio before it needs a slot.
RESUME_POLLS = 1
PARK_POLLS = 4


class LivePlan(NamedTuple):
    park: list  # running requests that give up their slot now
    resume: list  # parked requests that get a slot, in this order, before any admission
    admit: list  # waiting requests in admission order (as many as may be admitted)
    fill: list  # parked requests for slots that are still free after the admissions


def schedule_live(running: Sequence[SlotRequest], parked: Sequence[SlotRequest], waiting: Sequence[SlotRequest],
                  now: float, slots: int, max_live: int, frames_per_poll: int) -> LivePlan:
    """Who runs for the next poll: a pure function of the requests and the clock.

    1. Only when no slot is free and a paced request below the resume threshold is parked or waiting: the running
       paced requests at or above the park threshold give up their slots, largest lead first, at most one per such
       candidate. An unpaced request is never parked.
    2. Parked requests below the resume threshold get slots, smallest lead first.
    3. Waiting requests are admitted while slots and `max_live` (running + parked) allow: overdue paced ones
       (negative lead) first, smallest lead first, then everything else in order of arrival.
    Slots still free after that go to parked requests, smallest lead first: a slot never idles while work exists."""
    resume_at, park_at = RESUME_POLLS * frames_per_poll, PARK_POLLS * frames_per_poll
    by_lead = lambda rs: sorted(rs, key=lambda r: r.lead(now))  # stable: ties keep their order
    due = by_lead(r for r in parked if r.lead(now) < resume_at)
    room = max_live - len(running) - len(parked)
    starting = [r for r in waiting if r.pace is not None and r.lead(now) < resume_at][:max(room, 0)]
    free = slots - len(running)
    park = []
    if free <= 0 and (due or starting):
        ahead = by_lead(r for r in running if r.pace is not None and r.lead(now) >= park_at)[::-1]
        park = ahead[:len(due) + len(starting)]
        free += len(park)
    resume = due[:max(free, 0)]
    free -= len(resume)
    overdue = by_lead(r for r in waiting if r.pace is not None and r.lead(now) < 0)
    order = overdue + [r for r in waiting if not (r.pace is not None and r.lead(now) < 0)]
    admit = order[:max(min(free, room), 0)]
    rest = [r for r in by_lead(parked) if not any(r is x for x in resume)]
    return LivePlan(park, resume, admit, rest)


def compact_moves(running: Sequence[int], free: Sequence[int], rows: int = STEP_ROWS) -> list:
    """(from slot, to slot) moves that put every running request into slots [0, rows): a pure function of the slots
    the running requests hold and the free ones. Only when all of them fit there (at most `rows` running): each one at
    or above `rows`, lowest first, goes to the lowest free slot below `rows`. Otherwise, or when none is above, no move.
    Every move goes downward."""
    running = sorted(int(s) for s in running)
    if len(running) > rows:
        return []
    high = [s for s in running if s >= rows]
    low = sorted(int(s) for s in free if int(s) < rows)
    return list(zip(high, low))


def kv_safe(avail: int, claims) -> bool:
    """Banker's rule over one resource, KV pages. `claims`: (need, alone) of every admitted request -- the pages it
    may still take before it ends, and the pages only its row maps now. Safe when the requests can be ordered so that
    each one's need fits in `avail` plus what those before it give back: a request that runs to its end takes its
    need and then returns it together with `alone`, a net gain of `alone`. Smallest need first finds such an order
    when one exists. A page shared with another row is not counted as returned, so a state called safe is safe."""
    for need, alone in sorted(claims, key=lambda c: (c[0], -c[1])):
        if need > avail:
            return False
        avail += alone
    return True


class ContinuousBatcher:
    def __init__(self, model, max_slots: int = 32, frames_per_poll: int = 8, min_free_to_admit: int = 1,
                 max_live: Optional[int] = None, clock: Callable[[], float] = time.monotonic, kv_growth: bool = False,
                 compact_rows: bool = False, fused_admission: bool = False):
        """`frames_per_poll`: decode frames between two looks at the device-side slot states (a finished slot
        idles for at most that many frames). `min_free_to_admit`: admissions wait until that many slots are
        free (or nothing is running) — every admission is one extra prefill pass + first frame that streams
        all weights for the new rows only, so grouping them trades admission latency for throughput. With
        `fused_admission` the first frame rides in the running frame and only the prefill pass is extra.
        `max_live`: the most requests admitted at a time, running plus parked; the default, `max_slots`, means
        nothing is ever parked. `clock`: the time source of the pacing policy (seconds).
        `kv_growth`: on an engine whose page pool cannot hold every request at its full budget, a request maps its
        prompt and one poll of frames at admission and takes further pages as it decodes, under the banker's rule
        (kv_safe); one that cannot get its next page now waits parked until it can. Off: prompt + budget are
        reserved at admission and a running request never waits (DESIGN.md §4b).
        `compact_rows`: each frame decodes rows [0, 1 + highest live slot) rather than all `max_slots`, and at a poll
        boundary, when the running requests fit in 32 rows, those in slots >= 32 move to the lowest free slots below 32
        (compact_moves; LmEngine.park_slot / resume_slot: a small state blob and a page-table row, no K/V copied). An
        engine of more than 32 slots then runs its 32-row step GEMMs, with the same bits. Off: every frame decodes
        all `max_slots` rows and a request never changes slot unless it is parked.
        `fused_admission`: an admitted request's prefill leaves its first frame (head, sampler, fast passes) to the
        poll's first decode frame, where it runs as one more row beside the running requests, instead of a frame of
        its own that streams the head and fast weights for the new rows alone; the tokens are the same, and the
        request makes `frames_per_poll` frames in its first poll instead of one more. Off: as before."""
        from .models.text2semantic.inference import _ensure_engine

        if not 1 <= max_slots <= MAX_DECODE_BATCH:
            raise ValueError(f"max_slots must be in 1..{MAX_DECODE_BATCH}")
        self.model = model
        self.cfg = model.config
        self.eng = _ensure_engine(model, max_slots)
        self.max_slots = max_slots
        self.max_live = max_slots if max_live is None else int(max_live)
        if self.max_live < max_slots:
            raise ValueError(f"max_live must be >= max_slots ({max_slots}), got {max_live}")
        self.clock = clock
        self.compact_rows = bool(compact_rows)
        self.fused_admission = bool(fused_admission)
        self._pending: set[int] = set()  # fused_admission: slots whose first frame the next decode frame runs
        self.moves = 0  # compact_rows: requests moved to a lower slot
        self.parked: list[SlotRequest] = []  # admitted, between two polls without a slot (SlotRequest._parked)
        self.frames_per_poll = int(frames_per_poll)
        self.min_free_to_admit = max(1, int(min_free_to_admit))
        self.waiting: list[SlotRequest] = []
        self.active: dict[int, SlotRequest] = {}
        self._len: dict[int, int] = {}  # slot -> upper bound of its context length
        self.frames_run = 0  # decode frames launched (each serves every active slot)
        self.slot_frames = 0  # sum over frames of the active slots (occupancy numerator)
        eng = self.eng
        eng.reset()
        getattr(eng, "_slot_tokens", {}).clear()  # idle rows of the frames below write position 0 of unused slots
        if hasattr(eng, "release_kv"):
            eng.release_kv()  # paged KV: unused slots map no page, so those writes go nowhere
        eng.set_slot_control(True)
        self._state = eng.buffer("slot_state")
        self._limit = eng.buffer("slot_limit")
        self._temp = eng.buffer("slot_temperature")
        self._top_p = eng.buffer("slot_top_p")
        self._top_k = eng.buffer("slot_top_k")
        self._seed = eng.buffer("slot_seed")
        self._n_out = eng.buffer("n_out")
        self._pos = eng.buffer("pos")
        self._ras = eng.buffer("ras_window")
        self._out = eng.buffer("out_tokens")
        pool = getattr(eng, "kv_pool", None)
        # growth only where page accounting is needed at all (the `paged` test of _admit)
        self.kv_growth = bool(kv_growth) and pool is not None and (
            pool.n_pages < pool.slots * pool.pages_per_slot or self.max_live > self.max_slots)
        self.short: list[SlotRequest] = []  # parked for pages (kv_growth), in the order they were parked
        self._kv = None  # kv_growth: (avail, {request: [need, alone]}) while one step is being scheduled
        if self.kv_growth:
            self._miss = eng.buffer("kv_miss")
            self._miss.zero_()
            # unused slots idle at position -1, as retired ones do: at position 0 over no page they would record a miss
            self._pos.fill_(-1)

    def close(self):
        """Give the engine back to the one-request-at-a-time entry points."""
        self.eng.set_slot_control(False)
        self.eng.reset()

    # ------------------------------------------------------------------------------------------
    def submit(self, req: SlotRequest) -> SlotRequest:
        """Queue a request. Everything that can be wrong with ONE request is rejected here, with a ValueError the
        caller can hand back to that request alone; what reaches the engine later cannot fail per request."""
        cfg = self.cfg
        p = req.prompt
        if not isinstance(p, torch.Tensor) or p.ndim != 2 or p.size(0) != cfg.num_codebooks + 1 or p.size(1) < 1:
            raise ValueError(f"prompt must be an integer tensor [{cfg.num_codebooks + 1}, T>=1], got "
                             f"{tuple(p.shape) if isinstance(p, torch.Tensor) else type(p)}")
        if p.is_floating_point() or p.dtype == torch.bool:
            raise ValueError(f"prompt must hold integer token ids / codes, got {p.dtype}")
        # the reference asserts 0 < top_p <= 1 and 0 < temperature < 2 (inference.py:541-542); top_k >= 1 keeps
        # rank 0 only at 1. The sampler materialises at most 256 ranks: a larger top_k behaves like 256.
        if not (0.0 < float(req.top_p) <= 1.0):
            raise ValueError(f"top_p must be in (0, 1], got {req.top_p}")
        if not (0.0 < float(req.temperature) < 2.0):
            raise ValueError(f"temperature must be in (0, 2), got {req.temperature}")
        if int(req.top_k) < 1:
            raise ValueError(f"top_k must be >= 1, got {req.top_k}")
        T = int(req.prompt.size(1))
        if T >= cfg.max_seq_len:  # inference.py:262-265
            raise ValueError(f"Input sequence length {T} exceeds max_seq_len {cfg.max_seq_len}")
        n = int(req.max_new_tokens) if req.max_new_tokens else cfg.max_seq_len - T
        n = min(n, cfg.max_seq_len - T, self.eng.max_frames, self.eng.kv_len - T)
        if n < 1:
            raise ValueError("no room for new tokens")
        pool = getattr(self.eng, "kv_pool", None)
        if pool is not None and kv_pages_for(T + n) > pool.n_pages:
            raise ValueError(f"{T} prompt rows + {n} frames need {kv_pages_for(T + n)} KV pages, more than the "
                             f"engine's whole pool of {pool.n_pages} (kv_pages)")
        if req.pace is not None:
            if not float(req.pace) > 0.0:
                raise ValueError(f"pace must be > 0 frames per second, got {req.pace}")
            if req.stream is None:
                req.stream = StreamClock()
        req._limit = n
        req._t_submit = self.clock()
        self.waiting.append(req)
        return req

    def idle(self) -> bool:
        return not self.waiting and not self.active and not self.parked and not self.short

    def _free_slots(self) -> list[int]:
        return [s for s in range(self.max_slots) if s not in self.active]

    def _park(self, req: SlotRequest):
        s = req.slot
        assert s not in self._pending, f"slot {s} is parked before its first frame"
        req._parked = self.eng.park_slot(s, self._len.pop(s))
        del self.active[s]
        req.slot = -1
        req.parks += 1
        self.parked.append(req)

    def _resume(self, req: SlotRequest, s: int):
        if any(r is req for r in self.short):
            self.short.remove(req)
            req.page_wait = max(req.page_wait, self.clock() - req._short_since)
        else:
            self.parked.remove(req)
        parked, req._parked = req._parked, None
        self.eng.resume_slot(s, parked)
        req.slot = s
        req.resumes += 1
        self.active[s] = req
        self._len[s] = parked.ctx_len

    def _move(self, req: SlotRequest, s: int):
        """Continue the running `req` in the free slot `s`: its per-slot state and page-table row go along, so it keeps
        its pages, RAS window, random stream and playback clock."""
        frm = req.slot
        parked = self.eng.park_slot(frm, self._len.pop(frm))
        del self.active[frm]
        self.eng.resume_slot(s, parked)
        req.slot = s
        self.active[s] = req
        self._len[s] = parked.ctx_len
        req.moves += 1
        self.moves += 1

    def _compact(self):
        for frm, to in compact_moves(list(self.active), self._free_slots()):
            if frm not in self._pending:  # a request waiting for its first frame stays in its slot
                self._move(self.active[frm], to)

    def _schedule(self):
        """One scheduling decision (schedule_live) carried out: park, resume, admit, fill. With kv_growth, requests
        parked for pages resume first, and every resume and admission needs a safe grant of its pages."""
        if self.kv_growth:
            self._kv = self._kv_state()
            self._grants = {}  # slot -> end granted to a request resumed in this step
            self._resume_short()
        plan = schedule_live(list(self.active.values()), self.parked, [] if self.short else self.waiting,
                             self.clock(), self.max_slots, self.max_live, self.frames_per_poll)
        for req in plan.park:
            self._park(req)
        free = self._free_slots()
        for req in plan.resume:
            if self.kv_growth:
                end = self._grant(req)
                if end is None:  # due, but short of pages: it waits with those parked for pages
                    self._to_short(req)
                    continue
                self._grants[free[0]] = end
            self._resume(req, free.pop(0))
        self._admit(plan.admit)
        free = self._free_slots()
        for req in plan.fill:
            if not free:
                break
            if self.kv_growth:
                end = self._grant(req)
                if end is None:
                    continue
                self._grants[free[0]] = end
            self._resume(req, free.pop(0))

    # ---- KV growth (kv_growth) -------------------------------------------------------------------------------------
    def _kv_state(self):
        """(pages available, {request: [need, alone]}) over every admitted request, running or parked."""
        pool = self.eng.kv_pool
        claims = {}
        for r in [*self.active.values(), *self.parked, *self.short]:
            held, alone = pool.row_pages(pool.table[r.slot] if r._parked is None else r._parked.row)
            claims[r] = [kv_pages_for(int(r.prompt.size(1)) + r._limit) - held, alone]
        return pool.available(), claims

    def _target(self, req: SlotRequest) -> int:
        """Positions `req` has mapped once the next poll's frames are written: they write from its next position,
        context length - 1, on; never past prompt + budget."""
        ctx = self._len[req.slot] if req._parked is None else req._parked.ctx_len
        return min(ctx - 1 + self.frames_per_poll, int(req.prompt.size(1)) + req._limit)

    def _grant(self, req: SlotRequest) -> Optional[int]:
        """The end of `req`'s next poll (_target) when the pages it takes leave the state safe (they are counted as
        taken from then on), else None."""
        pool = self.eng.kv_pool
        end = self._target(req)
        held, _ = pool.row_pages(pool.table[req.slot] if req._parked is None else req._parked.row)
        g = kv_pages_for(end) - held
        if g <= 0:
            return end
        avail, claims = self._kv
        need, alone = claims[req]
        trial = dict(claims)
        trial[req] = [need - g, alone + g]
        if g > avail or not kv_safe(avail - g, trial.values()):
            return None
        claims[req] = trial[req]
        self._kv = (avail - g, claims)
        return end

    def _resume_short(self):
        """Requests parked for pages take free slots, in FIFO order, each once its grant is safe. One whose grant is not
        safe yet lets the next one try: the first request of the safe order may be behind it."""
        free = self._free_slots()
        for req in list(self.short):
            if not free:
                break
            end = self._grant(req)
            if end is not None:
                self._resume(req, free.pop(0))
                self._grants[req.slot] = end

    def _to_short(self, req: SlotRequest):
        self.parked.remove(req)
        self.short.append(req)
        req.page_parks += 1
        req._short_since = self.clock()

    def _grow(self):
        """Pages for the positions the next poll writes, for every running request, granted in safety order (smallest
        need first); a request whose grant would make the state unsafe is parked for pages before the frames run.
        One page-table upload for all grants (LmEngine.grow_kv)."""
        ends, short = dict(self._grants), []
        claims = self._kv[1]
        # a request admitted with its first frame pending holds its first poll's pages from admission: nothing to grant
        for req in sorted((r for r in self.active.values() if r.slot not in ends and r.slot not in self._pending),
                          key=lambda r: claims[r][0]):
            end = self._grant(req)
            if end is None:
                short.append(req)
            else:
                ends[req.slot] = end
        for req in short:
            self._park(req)
            self._to_short(req)
        if short:  # the slots they left may serve a request parked for pages whose grant is safe
            self._resume_short()
            ends.update(self._grants)
        self.eng.grow_kv(ends)
        self._kv = None

    def cancel(self, req: SlotRequest) -> bool:
        """Take `req` out wherever it is: waiting, running or parked. A running request's slot idles from the next
        frame on and its pages stay a reusable prefix, as after a normal end; a parked one's pages go back to the
        pool. `req.error` becomes a `Cancelled`, `done` / `on_done` fire; the other requests are unaffected.
        False when the request is already done (or was never submitted here)."""
        if req.done.is_set():
            return False
        if any(r is req for r in self.waiting):
            self.waiting.remove(req)
        elif self.active.get(req.slot) is req:
            self._vacate([req])
        elif req._parked is not None and any(r is req for r in self.parked + self.short):
            (self.short if any(r is req for r in self.short) else self.parked).remove(req)
            parked, req._parked = req._parked, None
            self.eng.drop_parked(parked)
        else:
            return False
        req.error = Cancelled("the request was cancelled")
        req.done.set()
        if req.on_done is not None:
            req.on_done(req)
        return True

    def _vacate(self, reqs: list, cache: bool = True):
        """The slots of `reqs` idle from the next frame on; their pages stay mapped as a reusable prefix (with the
        engine's prefix cache: their prompts' pages are cached, unless `cache` is False)."""
        idx = torch.tensor([r.slot for r in reqs], dtype=torch.long, device=self._state.device)
        self._state[idx] = 0
        self._pos[idx] = -1  # parked: the decode frames neither attend for this row nor touch its K/V (which a
        #                      later request with the same prompt prefix may reuse)
        for r in reqs:
            del self.active[r.slot]
            del self._len[r.slot]
            self._pending.discard(r.slot)  # a first frame still pending is dropped with the slot's state
            if not hasattr(self.eng, "retire_slot"):
                continue
            if cache:
                self.eng.retire_slot(r.slot)  # its pages stay a reusable prefix until the pool needs them
            else:
                self.eng.retire_slot(r.slot, cache=False)  # its tokens are void: its prompt is not cached

    def _admit(self, order: Optional[list] = None):
        """Admit the requests of `order` (from `waiting`; default: as they arrived), in that order, into free slots."""
        order = list(self.waiting) if order is None else order
        free = self._free_slots()
        if not free or not order:
            return
        if self.active and len(free) < min(self.min_free_to_admit, len(self.waiting)):
            return
        batch, slots = [], []
        budget = self.eng.max_rows  # one prefill pass worth of rows per step keeps decode latency bounded
        pool = getattr(self.eng, "kv_pool", None)
        # a pool with room for every slot at full capacity never runs out, unless parked requests hold pages beside
        # the slots' own: otherwise no page accounting is needed
        paged = pool is not None and (pool.n_pages < pool.slots * pool.pages_per_slot or self.max_live > self.max_slots)
        pages = self.eng.kv_pages_available() if paged else 0
        for head in order:
            if not free:
                break
            T = int(head.prompt.size(1))
            if batch and T > budget:
                break
            if paged:
                # FIFO: the head of the queue waits until its pages fit, and nothing overtakes it
                if head.reuse_prefix and head._host_prompt is None:  # one device -> host copy per request
                    head._host_prompt = head.prompt.detach().to("cpu", torch.int32)
                end = T + (min(self.frames_per_poll, head._limit) if self.kv_growth else head._limit)
                need = self.eng.kv_pages_needed(head._host_prompt, end, free[0], busy=slots, reuse=head.reuse_prefix)
                if self.kv_growth:
                    # growth: it maps its prompt and one poll of frames, if the state with it admitted is safe (it is
                    # counted as giving nothing back: its prefix may be shared)
                    avail, claims = self._kv
                    claim = [kv_pages_for(T + head._limit) - kv_pages_for(end), 0]
                    if need > avail or not kv_safe(avail - need, [*claims.values(), claim]):
                        break
                    claims[head] = claim
                    self._kv = (avail - need, claims)
                elif need > pages:
                    break
                pages -= need
            req = head
            self.waiting.remove(req)
            s = free.pop(0)
            req.slot = s
            batch.append(req)
            slots.append(s)
            budget -= T
        if not batch:
            return
        idx = torch.tensor(slots, dtype=torch.long, device=self._state.device)

        def put(buf, vals, dtype):
            buf[idx] = torch.tensor(vals, dtype=dtype, device=buf.device)

        put(self._limit, [r._limit for r in batch], torch.int32)
        put(self._temp, [bf16_round(r.temperature) for r in batch], torch.float32)
        put(self._top_p, [bf16_round(r.top_p) for r in batch], torch.float32)
        put(self._top_k, [int(r.top_k) for r in batch], torch.int32)
        put(self._seed, [int(r.seed) & 0x7FFFFFFFFFFFFFFF for r in batch], torch.int64)
        self._n_out[idx] = 0
        self._ras[idx] = 0
        self._state[idx] = 1
        for r in batch:
            self.active[r.slot] = r
            self._len[r.slot] = int(r.prompt.size(1)) + 1
        self.eng.set_context_bound_exact(max(self._len.values()) + 1)
        # paged KV: every request's pages (prompt + budget) are reserved before its prefill
        # (with kv_growth: the prompt and the first poll's frames)
        kw = dict(kv_end=[int(r.prompt.size(1)) + (min(self.frames_per_poll, r._limit) if self.kv_growth else r._limit)
                          for r in batch]) if pool is not None else {}
        if self.fused_admission:  # the first frames run in the next decode frame (_len above stays an upper bound)
            kw["defer_first_frame"] = True
            self._pending.update(slots)
        if any(r.reuse_prefix for r in batch) and hasattr(self.eng, "prefill_reusing"):
            self.eng.prefill_reusing([r.prompt for r in batch], slots, None, do_sample=True, **kw)
        else:
            self.eng.prefill([r.prompt for r in batch], slots, None, do_sample=True, **kw)

    def _retire(self) -> list[SlotRequest]:
        rows = [self._state.to(torch.int32), self._n_out] + ([self._miss] if self.kv_growth else [])
        st = torch.stack(rows).cpu()  # one small D2H copy (synchronises)
        if self.kv_growth:
            self._fail_missed(st[2])
        for s, req in self.active.items():
            # frames of a streaming request leave as soon as they are final: all but the newest one (the last frame of
            # a request -- <|im_end|> or the one at the budget -- is never part of what generate_long keeps)
            if req.on_frames is None and req.stream is None:
                continue
            n = int(st[1, s])
            if n - 1 > req._emitted:
                if req.on_frames is not None:
                    req.on_frames(req, self._out[s, 1:, req._emitted: n - 1].cpu())
                if req.stream is not None:  # the playback clock starts with the first frames handed out
                    if req.stream.t_first is None:
                        req.stream.t_first = self.clock()
                    req.stream.frames += n - 1 - req._emitted
                req._emitted = n - 1
        finished = []
        for s, req in list(self.active.items()):
            if int(st[0, s]) != 2:
                continue
            n = int(st[1, s])
            gen = self._out[s, :, :n].to(req.prompt.dtype)
            req.result = torch.cat([req.prompt.to(gen.device), gen], dim=1)
            finished.append(req)
        if finished:
            self._vacate(finished)
        for req in finished:
            req.done.set()
            if req.on_done is not None:
                req.on_done(req)
        return finished

    def _fail_missed(self, miss: torch.Tensor):
        """Requests whose decode attention met an unmapped page (the "kv_miss" buffer) sampled from a void attention:
        each fails alone, with the slot and position; its neighbours continue."""
        bad = [r for s, r in self.active.items() if int(miss[s]) != 0]
        if not bad:
            return
        for r in bad:
            r.error = RuntimeError(f"slot {r.slot}: decode attention met an unmapped KV page at position "
                                   f"{int(miss[r.slot]) - 1}; the request's tokens are void")
        self._miss[torch.tensor([r.slot for r in bad], dtype=torch.long, device=self._miss.device)] = 0
        self._vacate(bad, cache=False)
        for r in bad:
            r.done.set()
            if r.on_done is not None:
                r.on_done(r)

    def step(self) -> list[SlotRequest]:
        """Park / resume paced requests and admit waiting ones into free slots (schedule_live), run
        `frames_per_poll` frames, retire what finished."""
        self._schedule()
        if self.kv_growth:
            self._grow()
        if not self.active:
            return []
        if self.compact_rows:
            self._compact()  # after the grants: a moved request takes the pages granted to its row along
        k = self.frames_per_poll
        for s in self._len:
            self._len[s] += k
        self.eng.set_context_bound_exact(min(max(self._len.values()) + 1, self.eng.kv_len))
        # every slot row is decoded: idle and frozen rows cost one attention position and nothing else
        # (the GEMMs stream the weights once for the engine's 32- or 64-row tile whatever the number of live rows);
        # compact_rows: only rows up to the highest live slot, on the 32-row tile when that is at most 32 rows
        rows = 1 + max(self.active) if self.compact_rows else self.max_slots
        self.eng.decode(rows, k, None, use_graph=True)
        self._pending.clear()
        self.frames_run += k
        self.slot_frames += k * len(self.active)
        return self._retire()

    def run(self) -> None:
        while not self.idle():
            self.step()
