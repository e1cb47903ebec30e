"""The exact models and emulations of tests/frame_ref.py on the CPU: test_frame_tail_gpu.py holds the kernels to them."""
from __future__ import annotations

import torch

from oracle import lm_oracle as O
from tests import frame_ref as F
from tests.kernel_ref import embed_ref, rbf


def _cfg(**over):
    return O.tiny_config(**over)


def test_embed_emul_matches_the_oracle_and_its_roundings():
    for scale in (True, False):
        cfg = _cfg(scale_codebook_embeddings=scale)
        w = O.make_weights(cfg, seed=3)
        emb, cb = w["embeddings.weight"], w["codebook_embeddings.weight"]
        C, cs, sb, se = cfg.num_codebooks, cfg.codebook_size, cfg.semantic_begin_id, cfg.semantic_end_id
        g = torch.Generator().manual_seed(1)
        tok = torch.randint(0, cs, (12, C + 1), generator=g)
        tok[:, 0] = torch.tensor([sb - 1, sb, se, se + 1, -3, cfg.vocab_size + 9, sb + 5, sb + 6, 0, 7, sb + 1, se])
        tok[6, 1], tok[7, C] = -4, cs + 11  # codes outside [0, cs) on semantic rows
        x = F.embed_emul(tok, emb, cb, C, cs, sb, se, scale)
        # by hand, row by row: the clamps, the codebook sum rounded once, the division on semantic rows only
        for i in range(tok.shape[0]):
            t = int(tok[i, 0])
            sem = sb <= t <= se
            e = emb[min(max(t, 0), cfg.vocab_size - 1)].float()
            if sem:
                s = torch.zeros_like(e)
                for c in range(C):
                    s = s + cb[c * cs + min(max(int(tok[i, c + 1]), 0), cs - 1)].float()
                v = rbf(e + rbf(s))
                if scale:
                    v = rbf(v / torch.tensor(float(C + 1)).sqrt())
            else:
                v = e
            assert torch.equal(x[i], v), f"row {i} (token {t})"
        # inside embed_ref's float64 bracket, whose centre is oracle.embed on the clamped ids
        lo, hi, mid, x64 = embed_ref(tok, emb, cb, C, cs, sb, se, scale)
        assert ((x >= lo) & (x <= hi)).all()
        cl = tok.clone()
        cl[:, 0] = cl[:, 0].clamp(0, cfg.vocab_size - 1)
        cl[:, 1:] = cl[:, 1:].clamp(0, cs - 1)
        st = O.LMState(cfg, {k: w[k].double() for k in ("embeddings.weight", "codebook_embeddings.weight")})
        assert torch.allclose(O.embed(st, cl[:, :, None])[:, 0], x64, rtol=0, atol=1e-12)
        # the emulation is not the float64 value rounded once: a two-rounding chain differs somewhere
        assert not torch.equal(x, rbf(x64))


def test_restricted_head_tied_and_untied():
    for tied in (True, False):
        cfg = _cfg(tie_word_embeddings=tied)
        w = O.make_weights(cfg, seed=4)
        W = F.restricted_head(w, cfg)
        src = w["embeddings.weight"] if tied else w["output.weight"]
        n_sem = cfg.semantic_end_id - cfg.semantic_begin_id + 1
        assert W.shape == (n_sem + 1, cfg.dim)
        assert torch.equal(W[0], src[cfg.semantic_begin_id]) and torch.equal(W[n_sem - 1], src[cfg.semantic_end_id])
        assert torch.equal(W[-1], src[cfg.im_end_id])
        # the head the reference keeps selectable: logits of these rows equal the full head's at the same ids
        x = torch.randn(3, cfg.dim).bfloat16()
        full = x.double() @ src.double().T
        ids = list(range(cfg.semantic_begin_id, cfg.semantic_end_id + 1)) + [cfg.im_end_id]
        assert torch.equal(x.double() @ W.double().T, full[:, ids])


def _state(B=8, C1=5, T=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    return dict(cur=torch.randint(0, 99, (B, C1), generator=g).int(), out=torch.full((B, C1, T), -1, dtype=torch.int32),
                n_out=torch.zeros(B, dtype=torch.int32), pos=torch.arange(B, dtype=torch.int32) + 10,
                state=torch.ones(B, dtype=torch.int32), limit=torch.full((B,), 100, dtype=torch.int32),
                step=torch.tensor([5], dtype=torch.int64))


def _end(s, rows, **kw):
    return F.frame_end_model(s["cur"], s["out"], s["n_out"], s["pos"], s["state"], s["limit"], s["step"], rows, **kw)


def test_frame_end_model_rules():
    s = _state()
    s["state"] = torch.tensor([0, 1, 2, 3, 1, 1, 1, 1], dtype=torch.int32)
    s["n_out"] = torch.tensor([0, 0, 0, 2, 3, 4, 9, 1], dtype=torch.int32)
    s["limit"] = torch.tensor([9, 9, 9, 9, 9, 9, 20, 2], dtype=torch.int32)
    out, n_out, pos, state, step = _end(s, 8)
    assert int(step) == 6
    assert n_out.tolist() == [0, 1, 0, 3, 4, 5, 10, 2]  # idle and finished slots are skipped
    assert state.tolist() == [0, 1, 2, 2, 1, 1, 1, 2]  # <|im_end|> and the limit freeze
    assert pos.tolist() == [10, 12, 12, 13, 15, 16, 17, 17]  # frozen slots keep their position
    assert torch.equal(out[1, :, 0], s["cur"][1]) and torch.equal(out[4, :, 3], s["cur"][4])
    assert (out[5] == -1).all() and (out[6] == -1).all(), "frames at or past T_cap are counted, not stored"
    assert (out[0] == -1).all() and (out[2] == -1).all()
    # without slot control every row is live and nothing freezes
    out, n_out, pos, state, _ = _end(s, 8, slot_control=False)
    assert n_out.tolist() == [1, 1, 1, 3, 4, 5, 10, 2] and torch.equal(state, s["state"])
    assert torch.equal(pos, s["pos"] + 1)
    # rows map to slots; rows past `rows` do nothing
    out, n_out, pos, _, _ = _end(s, 2, row_slot=torch.tensor([4, 1, 0], dtype=torch.int32))
    assert n_out.tolist() == [0, 1, 0, 2, 4, 4, 9, 1] and pos.tolist() == [10, 12, 12, 13, 15, 15, 16, 17]
    # the prefill tail: positions from the prefill's rows, + 1 unless frozen
    src = torch.tensor([50, 60, 70, 80], dtype=torch.int32)
    _, _, pos, _, _ = _end(s, 4, row_slot=torch.tensor([1, 3, 7, 0], dtype=torch.int32),
                           set_pos_rows=torch.tensor([2, 0, 3, 1], dtype=torch.int32), row_pos_src=src)
    assert pos.tolist() == [10, 71, 12, 50, 14, 15, 16, 80]  # slot 0 idle; slots 3 and 7 freeze


def test_splice_model_rules():
    B, D = 8, 16
    x = torch.zeros(B, D)
    ssq = torch.zeros(B, 32)
    pos = torch.arange(B, dtype=torch.int32)
    pending = torch.tensor([0, 0, 0, 0, 1, 1, 1, 1], dtype=torch.int32)
    state = torch.tensor([0, 1, 2, 3, 0, 1, 2, 3], dtype=torch.int32)
    sx, sssq = torch.ones(B, D), torch.full((B, 32), 2.0)
    spos = torch.arange(B, dtype=torch.int32) + 100
    nx, nssq, npos, npend = F.splice_model(x, ssq, pos, pending, state, sx, sssq, spos, B)
    copied = [5, 7]
    for r in range(B):
        assert bool((nx[r] == 1).all()) == (r in copied) and bool((nssq[r] == 2).all()) == (r in copied)
    assert npos.tolist() == [0, 1, 2, 3, 4, 105, 6, 107]
    assert npend.tolist() == [0] * B
    _, _, _, npend = F.splice_model(x, ssq, pos, pending, state, sx, sssq, spos, 6)
    assert npend.tolist() == [0, 0, 0, 0, 0, 0, 1, 1], "rows past `rows` keep their flag"
