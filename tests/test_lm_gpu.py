"""Dual-AR engine (CUDA, through the C-ABI) against the oracle and against the committed outputs of
the real reference.

Tolerances: integer results (token ids / codebook indices) must be IDENTICAL wherever the oracle's
decision is not a near-tie; logits are bf16 values of fp32 sums accumulated in a different order than
the CPU's, so they are compared with atol = 2 bf16 ulps of the largest logit + 3% of the logit std.
"""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import lm_oracle as O
from tests.lm_util import (assert_tokens_match, build_model, load_golden, make_prompt, restricted,
                            teacher_forced_check)

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"


def _logit_tol(ref: torch.Tensor) -> float:
    return float(ref.abs().max()) * 2 ** -7 + 0.03 * float(ref.std())


def _gen(model, prompt, n, **kw):
    from fish_speech_b200.models.text2semantic.inference import generate

    return generate(model=model, prompt=prompt.cuda(), max_new_tokens=n, **kw).cpu()


@pytest.mark.parametrize("name", sorted(p.name for p in GOLD.glob("lm_*.npz") if int(np.load(p)["top_k"]) == 1))
def test_greedy_tokens_match_reference_golden(name):
    """Free-running greedy decode: every token id and codebook index equals the reference's."""
    cfg, w, z = load_golden(GOLD / name)
    model = build_model(cfg, w)
    got = _gen(model, torch.from_numpy(z["prompt"]), int(z["new_frames"]), temperature=float(z["temperature"]),
               top_p=float(z["top_p"]), top_k=int(z["top_k"]))
    ref = torch.from_numpy(z["ref_tokens"])
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert torch.equal(got.to(torch.int32), ref), f"first mismatch at {(got != ref).nonzero()[:4].tolist()}"


def _reference_uniforms(cfg, rng_seed: int, frames: int, head_rows: int) -> torch.Tensor:
    """The uniforms torch.rand produced during the recorded reference run, in the reference's order
    (multinomial_sample_one_no_sync, inference.py:43-46, called by sample() :86-93): per frame one [vocab] draw for
    the main token, one [vocab] draw for the RAS re-draw (:114-131, drawn even when unused), then one
    [codebook_size] draw per fast codebook 1..C-1 (:160-174); all in the probs dtype (bf16).  Laid out as the
    sampler hook expects: [frame][2 * draw_id + which][restricted candidate]."""
    C = cfg.num_codebooks
    u = torch.full((frames, 2 * C, max(head_rows, cfg.codebook_size)), 0.5)
    torch.manual_seed(rng_seed)
    for f in range(frames):
        for d in (0, 1):
            r = torch.rand(cfg.vocab_size, dtype=torch.bfloat16).float()
            u[f, d, : head_rows - 1] = r[cfg.semantic_begin_id: cfg.semantic_end_id + 1]
            u[f, d, head_rows - 1] = r[cfg.im_end_id]
        for p in range(1, C):
            u[f, 2 * p, : cfg.codebook_size] = torch.rand(cfg.codebook_size, dtype=torch.bfloat16).float()
    return u


def _stored_traces(path, frames: int) -> list:
    z = np.load(path)
    out = []
    for f in range(frames):
        scores, r = [], 0
        while f"s_{f}_{r}" in z.files:
            scores.append((torch.from_numpy(z[f"s_{f}_{r}"]), torch.from_numpy(z[f"cum_{f}_{r}"]), float(z[f"tp_{f}_{r}"]),
                           torch.from_numpy(z[f"topl_{f}_{r}"])))
            r += 1
        out.append({"scores": scores, "ras_changed": bool(z["ras_changed"][f])})
    return out


@pytest.mark.parametrize("name", ["lm_tiny_topk.npz", "lm_tiny_ras.npz"])
def test_stochastic_decode_replays_reference_rng(name):
    """top-k / top-p / temperature sampling AND the RAS substitution, bit-exact: the sampler is fed the very
    uniforms torch's generator produced in the recorded run of the real reference (debug hook
    fsb_lm_set_sampler_noise) and must emit the reference's token ids and codes for every frame.
    lm_tiny_ras repeats tokens inside the 10-frame window, so the high-temperature re-draw replaces the main
    token in >= 5 frames (stored in the fixture)."""
    cfg, w, z = load_golden(GOLD / name)
    model = build_model(cfg, w)
    eng = model.engine
    n = int(z["new_frames"])
    if "ras" in name:
        assert int(z["ras_changed"]) >= 5
    eng.set_sampler_noise(_reference_uniforms(cfg, int(z["rng_seed"]), n, eng.head_rows))
    try:
        got = _gen(model, torch.from_numpy(z["prompt"]), n, temperature=float(z["temperature"]),
                   top_p=float(z["top_p"]), top_k=int(z["top_k"]))
    finally:
        eng.set_sampler_noise(None)
    ref = torch.from_numpy(z["ref_tokens"])
    T = z["prompt"].shape[1]
    got = got.to(torch.int32)
    # The reference takes argmax(probs / q) over BF16 tensors: with an 8-bit mantissa two candidates' scores are often
    # equal or one ulp apart, and one ulp is also what a different (but correct) fp32 summation order inside a softmax
    # moves a bf16 probability by. A frame may differ only where the reference's own decision was such a near-tie
    # (top-2 scores within 2 bf16 ulps; or a sorted cumulative probability within 2 ulps of top_p, so that the top-p cut
    # keeps one candidate more or less; or the logits on either side of the top-k cut closer than the logit tolerance
    # of this suite, so that another candidate enters the top k -- all taken from the oracle's trace of the same run);
    # the runs then follow different histories, so the comparison stops there. Everything before must be identical,
    # RAS substitutions included.  The oracle's trace is stored with the golden (oracle/make_golden_traces.py, recorded
    # where the oracle reproduces the reference run exactly): its CPU bf16 matmuls depend on the host's instruction set.
    traces = _stored_traces(GOLD / ("trace_" + name), n)
    frames_equal, ras_verified = 0, 0
    for f in range(n):
        if T + f >= got.shape[1] or T + f >= ref.shape[1]:
            break
        if torch.equal(got[:, T + f], ref[:, T + f]):
            frames_equal += 1
            ras_verified += bool(traces[f].get("ras_changed"))
            continue
        r = int((got[:, T + f] != ref[:, T + f]).nonzero()[0])
        sc = traces[f]["scores"]
        cand = [sc[0], sc[1]] if r <= 1 else [sc[r]]  # row 0/1: main token (or its RAS re-draw); row r >= 2: codebook r-1
        gaps = []
        for s_, cum, tp, topl in cand:
            top2 = torch.topk(s_[torch.isfinite(s_)], 2).values
            gaps.append(float(top2[0] - top2[1]) / (float(top2[0].abs()) * 2 ** -7 + 1e-30))
            gaps.append(float((cum - tp).abs().min()) / (tp * 2 ** -7))
            if topl.numel() > int(z["top_k"]):  # top-k cut: 2.0 on this scale = the logit tolerance (_logit_tol)
                gaps.append(2.0 * float(topl[-2] - topl[-1]) / _logit_tol(topl))
        assert min(gaps) <= 2.0, (f"frame {f} row {r}: got {got[:, T + f].tolist()} want {ref[:, T + f].tolist()}; the reference's "
                                  f"decision was not a near-tie (score / top-p-cut / top-k-cut gaps, 2.0 = tolerance: {[round(g, 2) for g in gaps]})")
        break
    else:
        assert got.shape == ref.shape
    print(f"{name}: {frames_equal}/{n} frames identical before the first bf16 score near-tie, {ras_verified} RAS substitutions verified")
    assert frames_equal >= 8, f"only {frames_equal} frames verified"
    if "ras" in name:
        assert ras_verified >= 3, f"only {ras_verified} RAS substitutions verified"


def test_prefill_and_decode_logits_teacher_forced():
    """Per-frame slow/fast logits vs the oracle with the oracle's own tokens fed back (teacher forcing)."""
    from fish_speech_b200.models.text2semantic.inference import decode_one_token_ar

    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=21, head_gain=4.0)
    st = O.setup(cfg, w)
    T, n = 11, 6
    prompt = make_prompt(cfg, 21, T)
    traces = []
    ref = O.generate(st, prompt, n, temperature=0.7, top_p=0.7, top_k=1, traces=traces, stop_on_im_end=False,
                     noise=False)
    model = build_model(cfg, w)
    eng = model.engine
    temp, top_p = torch.tensor(0.7), torch.tensor(0.7)
    C1 = cfg.num_codebooks + 1
    prev = torch.zeros((C1, 10), dtype=torch.int32)
    for f in range(n):
        if f == 0:
            x, pos, pt = prompt.view(1, C1, -1).cuda(), torch.arange(T).cuda(), None
        else:
            x = ref[:, T + f - 1].view(1, C1, 1).cuda()  # the ORACLE's previous frame
            pos, pt = torch.tensor([T + f - 1]).cuda(), prev.cuda()
        tok = decode_one_token_ar(model, x, pos, temp, top_p, 1, None, None, None, previous_tokens=pt).cpu()
        slow = eng.buffer("slow_logits")[0].cpu()
        want = restricted(cfg, traces[f]["slow_logits"])
        tol = _logit_tol(want)
        assert (slow - want).abs().max().item() <= tol, f"frame {f}: slow logits off by {(slow - want).abs().max().item()} > {tol}"
        fast = eng.buffer("fast_logits")[: cfg.num_codebooks - 1, 0].cpu()
        # fast logits depend on the sampled codes: compare only while our codes equal the oracle's
        same = torch.equal(tok.view(-1).to(torch.int32), ref[:, T + f].to(torch.int32))
        assert same, f"frame {f}: tokens {tok.view(-1).tolist()} vs oracle {ref[:, T + f].tolist()}"
        for p in range(cfg.num_codebooks - 1):
            wantf = traces[f]["fast_logits"][p]
            assert (fast[p] - wantf).abs().max().item() <= _logit_tol(wantf), f"frame {f} fast pass {p + 1}"
        if f > 0:
            prev = prev.roll(-1, dims=1)
            prev[:, -1] = ref[:, T + f].to(torch.int32)


def test_batch_invariance_and_ragged_prompts():
    """Batch-32-style decode: each sequence of a ragged batch equals its solo run and the oracle."""
    from fish_speech_b200.models.text2semantic.inference import generate_batch

    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=31, head_gain=8.0)
    lens = [5, 17, 9, 30, 12]
    prompts = [make_prompt(cfg, 100 + i, T) for i, T in enumerate(lens)]
    n = 9
    model = build_model(cfg, w, max_batch=len(lens))
    outs = generate_batch(model=model, prompts=[p.cuda() for p in prompts], max_new_tokens=n, temperature=0.7,
                          top_p=0.7, top_k=1)
    solo = build_model(cfg, w, max_batch=1)
    for i, p in enumerate(prompts):
        one = _gen(solo, p, n, temperature=0.7, top_p=0.7, top_k=1)
        assert torch.equal(outs[i].cpu().to(torch.int32), one.to(torch.int32)), f"seq {i}: batch != solo"
        eq, ties, dec = teacher_forced_check(solo, cfg, w, p, n, f"seq {i}")
        assert dec >= 0.6 * n * cfg.num_codebooks, f"seq {i}: {eq}/{n} frames identical, {ties} near-ties, {dec} decisions"


class _PrefillCalls:
    """Stands in for an engine's library handle and counts its fsb_lm_prefill calls (one per prefill pass)."""

    def __init__(self, lib):
        self._lib, self.calls = lib, 0

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if name != "fsb_lm_prefill":
            return f

        def counted(*args):
            self.calls += 1
            return f(*args)
        return counted


def test_prefill_chunking_equals_single_pass():
    """max_rows smaller than the prompt: a 150-row prompt prefilled 48 rows at a time (pieces start at 48, 96 and 144,
    so the page edges at 64 and 128 fall inside pieces) must give the continuation of a single pass."""
    cfg = O.tiny_config(max_seq_len=256)
    w = O.make_weights(cfg, seed=41, head_gain=8.0)
    T = 150
    p = make_prompt(cfg, 41, T)
    passes = []
    for max_rows in (2048, 48):
        model = build_model(cfg, w, max_rows=max_rows)
        model.engine.lib = calls = _PrefillCalls(model.engine.lib)
        passes.append((_gen(model, p, 6, temperature=0.7, top_p=0.7, top_k=1), calls.calls))
        model.engine.close()
    (a, n_one), (b, n_chunked) = passes
    assert n_one == 1 and n_chunked == 4, f"prefill passes: {n_one} with max_rows 2048, {n_chunked} with 48"
    assert torch.equal(a, b)
    st = O.setup(cfg, w)
    traces = []
    ref = O.generate(st, p, 6, temperature=0.7, top_p=0.7, top_k=1, traces=traces, noise=False)
    assert_tokens_match(a, ref, traces, cfg, T, "chunked prefill")


def test_s2pro_layer_geometry_greedy():
    """S2-Pro layer shapes (dim 2560, 32/8 heads x 128, I 9728, 10 codebooks x 4096) with few layers and a
    reduced vocabulary so the CPU oracle finishes in seconds: greedy tokens identical."""
    cfg = O.LMConfig(n_layer=2, n_fast_layer=1, vocab_size=8192, max_seq_len=256, semantic_begin_id=4000,
                     semantic_end_id=8095, im_end_id=3999)
    w = O.make_weights(cfg, seed=51, head_gain=6.0)
    p = make_prompt(cfg, 51, 24)
    eq, ties, dec = teacher_forced_check(build_model(cfg, w), cfg, w, p, 6, "s2pro geometry")
    # 10 x 4096-way decisions per frame on random weights: ~15% of them are bf16 near-ties (top-2 gap
    # <= 2 ulp); every other decision must be identical (hard mismatches fail inside the helper)
    assert dec >= 30, f"only {dec}/60 decisions verified ({eq} frames identical, {ties} near-ties)"


def test_stop_on_im_end_and_max_len_errors():
    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=61, head_gain=8.0)
    p = make_prompt(cfg, 61, 10)
    # make <|im_end|> win at frame 3: give its head row 1.5x the row of the token a free run picks there
    free = O.generate(O.setup(cfg, w), p, 6, temperature=0.7, top_p=0.7, top_k=1, noise=False)
    w["embeddings.weight"][cfg.im_end_id] = (w["embeddings.weight"][int(free[0, 13])].float() * 1.5).bfloat16()
    st = O.setup(cfg, w)
    ref = O.generate(st, p, 20, temperature=0.7, top_p=0.7, top_k=1, noise=False)
    assert ref[0, -1].item() == cfg.im_end_id and ref.shape[1] <= 10 + 4
    model = build_model(cfg, w)
    got = _gen(model, p, 20, temperature=0.7, top_p=0.7, top_k=1)
    assert got.shape == ref.shape and torch.equal(got[0].to(torch.int32), ref[0])
    assert got.shape[1] < 10 + 20 and got[0, -1].item() == cfg.im_end_id
    with pytest.raises(ValueError):
        _gen(model, torch.zeros(cfg.num_codebooks + 1, cfg.max_seq_len, dtype=torch.long), 4)


def test_stochastic_sampling_distribution():
    """top-k / top-p / temperature sampling: empirical token frequencies of the first generated frame
    follow the oracle's logits_to_probs distribution (our Philox stream differs from torch's)."""
    from fish_speech_b200.models.text2semantic.inference import generate

    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=71, head_gain=2.5)
    p = make_prompt(cfg, 71, 8)
    st = O.setup(cfg, w)
    logits, _ = O.forward_generate(st, p.view(1, cfg.num_codebooks + 1, -1), torch.arange(8))
    dt = torch.bfloat16
    probs = O.logits_to_probs((logits + O.semantic_logit_bias(cfg, dt))[0, -1], torch.tensor(0.9, dtype=dt),
                              torch.tensor(0.8, dtype=dt), 5).float()
    model = build_model(cfg, w)
    N = 600
    counts = torch.zeros(cfg.vocab_size)
    for s in range(N):
        out = generate(model=model, prompt=p.cuda(), max_new_tokens=1, temperature=0.9, top_p=0.8, top_k=5, seed=s)
        counts[int(out[0, 8].item())] += 1
    freq = counts / N
    support = probs > 0
    assert freq[~support].sum().item() == 0, "sampled a token outside the top-k/top-p support"
    assert (freq - probs).abs().max().item() < 0.08, (freq[support], probs[support])


def test_large_kv_capacity_small_context():
    """A checkpoint-sized max_seq_len (32768, the S2-Pro config value) must not size the attention score
    buffer: it follows the live context bound tracked by the host."""
    cfg = O.tiny_config(max_seq_len=32768)
    w = O.make_weights(cfg, seed=81, head_gain=8.0)
    p = make_prompt(cfg, 81, 20)
    ref_cfg = O.tiny_config(max_seq_len=128)  # same weights / tables for the positions touched
    traces = []
    ref = O.generate(O.setup(ref_cfg, w), p, 6, temperature=0.7, top_p=0.7, top_k=1, traces=traces, noise=False)
    got = _gen(build_model(cfg, w), p, 6, temperature=0.7, top_p=0.7, top_k=1)
    assert assert_tokens_match(got, ref, traces, ref_cfg, 20, "kv capacity 32768") >= 4


def test_frame_callback_streams_exactly_the_kept_codes():
    """generate(frame_callback=...) hands out the codes of finished frames while decoding continues; the pieces
    concatenate to what generate_long keeps of the call, y[1:, T:-1] (inference.py:708), for a budget-limited run and
    for one that stops on <|im_end|>."""
    from fish_speech_b200.models.text2semantic.inference import generate

    cfg = O.tiny_config()
    p = make_prompt(cfg, 61, 10)

    def run(model):
        pieces = []
        y = generate(model=model, prompt=p.cuda(), max_new_tokens=20, temperature=0.7, top_p=0.7, top_k=1,
                     frame_callback=lambda b, codes: pieces.append(codes.clone()))
        kept = y[1:, 10:-1].cpu()
        got = torch.cat(pieces, dim=1) if pieces else kept[:, :0]
        assert all(c.device.type == "cpu" for c in pieces)
        assert torch.equal(got.to(kept.dtype), kept), (got.shape, kept.shape)
        if kept.shape[1] > 8:  # frames are handed out at every poll (8 frames), the newest one held back
            assert len(pieces) >= 2
        return y, pieces

    w = O.make_weights(cfg, seed=61, head_gain=8.0)
    w["embeddings.weight"][cfg.im_end_id] = 0  # a zero head row: <|im_end|> never wins, the budget ends the run
    y, pieces = run(build_model(cfg, w, debug=False))
    assert y.shape[1] == 30 and len(pieces) == 3
    # make <|im_end|> win somewhere in the run: its head row = 1.5 x the row of the token the free run picks at frame 11
    # (it stops at the first frame where that token would have won)
    w2 = dict(w)
    w2["embeddings.weight"] = w["embeddings.weight"].clone()
    w2["embeddings.weight"][cfg.im_end_id] = (w["embeddings.weight"][int(y[0, 10 + 11])].float() * 1.5).bfloat16()
    y, pieces = run(build_model(cfg, w2, debug=False))
    assert y[0, -1].item() == cfg.im_end_id and y.shape[1] < 30


def _rolled_layers(cfg: O.LMConfig, seed: int, head_gain: float) -> dict:
    """Full-size synthetic weights without drawing 4.5 G random numbers: layer l of a stack is layer 0's tensors rolled by
    l rows (every layer distinct, so a mixed-up layer index changes the result), embeddings / heads drawn once."""
    one = O.LMConfig(**{**cfg.__dict__, "n_layer": 1, "n_fast_layer": 1})
    w = O.make_weights(one, seed=seed, head_gain=head_gain)
    for stack, n in (("layers", cfg.n_layer), ("fast_layers", cfg.n_fast_layer)):
        base = {k: v for k, v in w.items() if k.startswith(f"{stack}.0.")}
        for l in range(1, n):
            for k, v in base.items():
                w[k.replace(f"{stack}.0.", f"{stack}.{l}.")] = torch.roll(v, shifts=l, dims=0) if v.ndim == 2 else v
    return w


def test_full_s2pro_geometry_batch32():
    """The real size: 36 + 4 layers at S2-Pro dimensions (dim 2560, 32/8 heads x 128, I 9728, 10 x 4096 codes, the 4097
    selectable head rows), batch 32 -- the benchmark's configuration. Sequences 0, 13 and 31 of the batch are checked
    against the CPU oracle run on each of them alone: token ids and codes identical up to the first decision the oracle
    itself took on a bf16 near-tie (random weights, 4096-way decisions). Vocabulary reduced to keep the CPU side short.
    Near-tie = oracle top-2 gap <= 6 x 2^-7 of the top logit here (2 x on the tiny models): through 36 layers of width
    2560 the two implementations' fp32 summation orders differ by more bf16 roundings of the residual stream; two
    revisions of the CUDA path that differ only in the attention's summation order flipped decisions at oracle gaps of
    2.2 and 3.7 x 2^-7 (4096-way decisions on random weights with head gain 6: logits around 20, bf16 ulp 0.125)."""
    from fish_speech_b200.models.text2semantic.inference import generate_batch

    cfg = O.LMConfig(vocab_size=8192, max_seq_len=128, semantic_begin_id=4000, semantic_end_id=8095, im_end_id=3999)
    w = _rolled_layers(cfg, seed=52, head_gain=6.0)
    prompts = [make_prompt(cfg, 500 + i, 20 + (i % 5)) for i in range(32)]
    model = build_model(cfg, w, max_batch=32, debug=False)
    outs = generate_batch(model=model, prompts=[p.cuda() for p in prompts], max_new_tokens=3, temperature=0.7, top_p=0.7,
                          top_k=1)
    st = O.setup(cfg, w)
    verified = 0
    for i in (0, 13, 31):
        traces = []
        ref = O.generate(O.setup(cfg, w) if i else st, prompts[i], 3, temperature=0.7, top_p=0.7, top_k=1, traces=traces,
                         stop_on_im_end=False, noise=False)
        T = prompts[i].shape[1]
        frames = assert_tokens_match(outs[i][:, : ref.shape[1]], ref, traces, cfg, T, f"full size, sequence {i}",
                                     tie_ulps=6.0)
        got, want = outs[i].cpu().to(torch.int32), ref.to(torch.int32)
        f = T + frames
        verified += frames * cfg.num_codebooks
        if f < want.shape[1]:  # decisions of the frame with the near-tie that precede it
            r = int((got[:, f] != want[:, f]).nonzero()[0])
            verified += max(0, r - 1)
    assert verified >= 20, f"only {verified} of 90 decisions verified before near-ties"
