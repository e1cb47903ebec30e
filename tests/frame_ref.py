"""Exact models and fp32 emulations of the launches of a decode frame around its two stacks (csrc/lm_engine.cu
frame_stage): the decode embed, the restricted slow head's weight, the first-frame splice and the frame end.
tests/test_frame_tail_gpu.py compares the kernels with them; tests/test_frame_tail_cpu.py rehearses them on the CPU.
Plain torch on whatever device the inputs live on."""
from __future__ import annotations

import torch

from tests.kernel_ref import rbf


def embed_emul(tokens, emb, cb_emb, C, cs, sem_begin, sem_end, scale):
    """embed_kernel in fp32: tokens int [rows][C+1] -> x fp32 [rows, D] holding bf16 values. The token decides
    'semantic' before it is clamped to [0, vocab); each code is clamped to [0, cs); a semantic row's codebook rows are
    summed in fp32 from 0 in codebook order and rounded to bf16 once; x = rbf(e + s) (s = 0 on other rows); semantic
    rows of a scaling model are then rbf(x / sqrtf(C + 1)) once more."""
    tok = tokens[:, 0].long()
    sem = (tok >= sem_begin) & (tok <= sem_end)
    e = emb[tok.clamp(0, emb.shape[0] - 1)].float()
    codes = tokens[:, 1:C + 1].long().clamp(0, cs - 1) + torch.arange(C, device=tokens.device)[None, :] * cs
    s = torch.zeros_like(e)
    for c in range(C):
        s = s + cb_emb[codes[:, c]].float()
    s = torch.where(sem[:, None], rbf(s), torch.zeros_like(s))
    x = rbf(e + s)
    if scale:
        div = torch.tensor(float(C + 1), dtype=torch.float32, device=x.device).sqrt()
        x = torch.where(sem[:, None], rbf(x / div), x)
    return x


def restricted_head(w, cfg, im_end_id=None):
    """The rows of the LM head the semantic logit bias leaves selectable (inference.py:308-320): the semantic ids in
    order, then <|im_end|>; the embedding matrix for a tied head, output.weight otherwise."""
    src = w["embeddings.weight"] if cfg.tie_word_embeddings else w["output.weight"]
    im = cfg.im_end_id if im_end_id is None else im_end_id
    return torch.cat([src[cfg.semantic_begin_id: cfg.semantic_end_id + 1], src[im: im + 1]], 0)


def splice_model(x, ssq, pos, pending, state, stage_x, stage_ssq, stage_pos, rows):
    """first_frame_splice_kernel: for each row r < rows (row r is slot r) whose first frame is pending, the staged row,
    its sums of squares and its position are copied in when the slot is live (state 1 or 3); the flag is cleared in
    every case. Returns new (x, ssq, pos, pending)."""
    x, ssq, pos, pending = x.clone(), ssq.clone(), pos.clone(), pending.clone()
    for r in range(rows):
        if int(pending[r]) == 0:
            continue
        if int(state[r]) in (1, 3):
            x[r] = stage_x[r]
            ssq[r] = stage_ssq[r]
            pos[r] = stage_pos[r]
        pending[r] = 0
    return x, ssq, pos, pending


def frame_end_model(cur_tok, out_tokens, n_out, pos, state, limit, step, rows, row_slot=None, slot_control=True,
                    set_pos_rows=None, row_pos_src=None):
    """frame_end_kernel + step_inc_kernel. For each row's slot (row i is slot row_slot[i], or i), when the slot is live
    (state 1 or 3; every slot without slot control): the frame's tokens go to out_tokens[slot][:, n_out] if
    n_out < T_cap (out_tokens' last dimension), n_out + 1, and the position advances by one unless the slot freezes
    (state 3, or n_out + 1 reaching its limit: state 2). With set_pos_rows, pos = row_pos_src[set_pos_rows[i]] (+ 1
    unless frozen) instead. step + 1 once. Returns new (out_tokens, n_out, pos, state, step)."""
    out_tokens, n_out, pos, state = out_tokens.clone(), n_out.clone(), pos.clone(), state.clone()
    T_cap = out_tokens.shape[-1]
    for i in range(rows):
        slot = int(row_slot[i]) if row_slot is not None else i
        if slot_control and int(state[slot]) not in (1, 3):
            continue
        f = int(n_out[slot])
        if f < T_cap:
            out_tokens[slot, :, f] = cur_tok[slot]
        n_out[slot] = f + 1
        advance = True
        if slot_control and (int(state[slot]) == 3 or f + 1 >= int(limit[slot])):
            state[slot] = 2
            advance = False
        if set_pos_rows is not None:
            pos[slot] = int(row_pos_src[int(set_pos_rows[i])]) + int(advance)
        elif advance:
            pos[slot] = pos[slot] + 1
    return out_tokens, n_out, pos, state, step + 1
