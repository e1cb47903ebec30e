"""Host side of the split decode attention (fsb_lm_config.attn_split): the ctypes mirror of the config, the validation
at fsb_lm_create (it runs before any device is looked for), setup_caches(attn_split=) and FSB_ATTN_SPLIT."""
import ctypes as C
import re
import time
from pathlib import Path

import pytest
import torch

from fish_speech_b200 import _lib
from fish_speech_b200.models.text2semantic import inference as inf
from fish_speech_b200.models.text2semantic import llama
from oracle import lm_oracle as O
from tests.lm_util import model_args
from tests.test_paged_kv_cpu import _S2ProSizedModel


def test_config_mirror_ends_with_attn_split():
    hdr = (Path(_lib.__file__).resolve().parent.parent / "include" / "fishb200.h").read_text()
    body = re.search(r"typedef struct \{(.*?)\} fsb_lm_config;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = [n.strip() for decl in re.findall(r"(?:int|float)\s+([^;]+);", body) for n in decl.split(",")]
    assert fields == [n for n, _ in _lib.LmConfig._fields_]
    assert fields[-1] == "attn_split"
    assert _lib.LmConfig().attn_split == 0  # off unless asked for


def _create(attn_split, **over):
    """fsb_lm_create on a config that is valid but for what the test sets; returns (rc, message)."""
    K = _lib.LmConfig()
    K.dim, K.n_layer, K.n_head, K.n_kv_head, K.head_dim, K.intermediate = 256, 1, 4, 1, 128, 512
    K.fast_dim, K.n_fast_layer, K.fast_n_head, K.fast_n_kv_head, K.fast_head_dim, K.fast_intermediate = 256, 1, 4, 1, 64, 512
    K.vocab_size, K.codebook_size, K.num_codebooks = 1200, 96, 4
    K.semantic_begin_id, K.semantic_end_id, K.im_end_id = 1000, 1095, 999
    K.max_batch, K.kv_len, K.max_rows, K.max_frames = 1, 32768, 128, 4
    K.attn_split = attn_split
    for k, v in over.items():
        setattr(K, k, v)
    W = _lib.LmWeights()
    W.head_rows = 97
    h = C.c_void_p()
    L = _lib.lib()
    rc = L.fsb_lm_create(C.byref(K), C.byref(W), C.byref(h))
    msg = L.fsb_last_error().decode()
    if rc == 0:
        L.fsb_lm_destroy(h)
    return rc, msg


@pytest.mark.parametrize("bad", [-64, 1, 100, 2047, 10944 + 64, 1 << 20])
def test_create_rejects_a_bad_attn_split(bad):
    rc, msg = _create(bad)
    assert rc != 0 and "attn_split" in msg and str(bad) in msg and "10944" in msg


def test_the_longest_span_follows_the_geometry():
    # 8 query heads per KV head: twice the scores per position, about half the span
    rc, msg = _create(8192, n_head=8)
    assert rc != 0 and "attn_split=8192" in msg and "[64, 5056]" in msg
    if not torch.cuda.is_available():  # a valid value gets past the validation: the next failure is the missing device
        rc, msg = _create(2048)
        assert rc != 0 and "attn_split" not in msg


def test_setup_caches_passes_attn_split_and_rebuilds_when_it_changes(monkeypatch):
    made = []

    class FakeEngine:
        def __init__(self, *a, **kw):
            made.append(kw)

        def close(self):
            pass

    monkeypatch.setattr(llama, "LmEngine", FakeEngine)
    cfg = O.tiny_config()
    m = llama.DualARTransformer(model_args(cfg), {}, device="cpu", im_end_id=cfg.im_end_id)
    m.setup_caches(max_batch_size=2, max_seq_len=128)
    m.setup_caches(max_batch_size=2, max_seq_len=128)
    m.setup_caches(max_batch_size=2, max_seq_len=128, attn_split=64)
    m.setup_caches(max_batch_size=2, max_seq_len=128, attn_split=64)
    assert [k["attn_split"] for k in made] == [0, 64] and m.attn_split == 64


def test_serve_attn_split_parses_the_variable():
    assert inf.serve_attn_split(None) == 0 and inf.serve_attn_split("") == 0 and inf.serve_attn_split("0") == 0
    assert inf.serve_attn_split("2048") == 2048
    for bad in ("-64", "100", "2k", "1.5"):
        with pytest.raises(ValueError, match="FSB_ATTN_SPLIT"):
            inf.serve_attn_split(bad)


@pytest.mark.parametrize("env,want", [(None, 0), ("4096", 4096)])
def test_serving_worker_hands_the_variable_to_setup_caches(monkeypatch, env, want):
    seen = []
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: (_S2ProSizedModel(), inf.decode_one_token_ar))
    monkeypatch.setattr(inf, "serve_requests", lambda model, q, slots: seen.append(model.caches))
    monkeypatch.setenv("FSB_SERVE_SLOTS", "64")
    monkeypatch.setenv("FSB_SERVE_KV_GB", "24")
    monkeypatch.delenv("FSB_SERVE_KV_LEN", raising=False)
    if env is None:
        monkeypatch.delenv("FSB_ATTN_SPLIT", raising=False)
    else:
        monkeypatch.setenv("FSB_ATTN_SPLIT", env)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (60 * 10 ** 9, 80 * 10 ** 9))
    inf.launch_thread_safe_queue("ckpt", "cuda", torch.bfloat16)
    for _ in range(200):
        if seen:
            break
        time.sleep(0.01)
    assert seen[0]["attn_split"] == want and seen[0]["kv_pages"] > 0


def test_serving_worker_reports_a_bad_variable(monkeypatch):
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: (_S2ProSizedModel(), inf.decode_one_token_ar))
    monkeypatch.setenv("FSB_SERVE_SLOTS", "8")
    monkeypatch.delenv("FSB_SERVE_KV_GB", raising=False)
    monkeypatch.setenv("FSB_ATTN_SPLIT", "1000")
    with pytest.raises(ValueError, match="FSB_ATTN_SPLIT"):
        inf.launch_thread_safe_queue("ckpt", "cpu", torch.bfloat16)
