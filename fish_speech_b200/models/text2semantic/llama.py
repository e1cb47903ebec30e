"""Drop-in surface of fish_speech/models/text2semantic/llama.py for the inference hot path.

Same names, config semantics, checkpoint formats and error behaviour as the reference
(`BaseModelArgs.from_pretrained` llama.py:75-143, `DualARModelArgs` :156-193, key remap :229-246,
`BaseTransformer.from_pretrained` :480-594, `setup_caches` :307-325/:708-721), but the model object
holds device weights plus a handle to the CUDA engine instead of nn.Modules: all math runs in
libfishb200.so.  Training-side features (forward with labels, LoRA, gradient checkpointing) are out of
scope (SURVEY.md §8).
"""
from __future__ import annotations

import dataclasses
import json
from collections import OrderedDict
from dataclasses import dataclass
from pathlib import Path
from typing import Iterator, Optional

import torch

from ...engine import LmEngine

IM_END_TOKEN = "<|im_end|>"  # fish_speech/tokenizer.py


def find_multiple(n: int, k: int) -> int:
    return n if n % k == 0 else n + k - (n % k)


@dataclass
class BaseModelArgs:
    model_type: str = "base"
    vocab_size: int = 32000
    n_layer: int = 32
    n_head: int = 32
    dim: int = 4096
    intermediate_size: int = None
    n_local_heads: int = -1
    head_dim: int = 64
    rope_base: float = 10000
    norm_eps: float = 1e-5
    max_seq_len: int = 2048
    dropout: float = 0.0
    tie_word_embeddings: bool = True
    attention_qkv_bias: bool = False
    attention_o_bias: bool = False
    attention_qk_norm: bool = False
    codebook_size: int = 160
    num_codebooks: int = 4
    semantic_begin_id: int = 0
    semantic_end_id: int = 0
    use_gradient_checkpointing: bool = True
    initializer_range: float = 0.02
    is_reward_model: bool = False
    scale_codebook_embeddings: bool = False
    audio_embed_dim: Optional[int] = None

    def __post_init__(self):
        if self.n_local_heads == -1:
            self.n_local_heads = self.n_head
        if self.intermediate_size is None:
            self.intermediate_size = find_multiple(int(2 * 4 * self.dim / 3), 256)
        if self.head_dim is None:
            self.head_dim = self.dim // self.n_head

    @staticmethod
    def from_pretrained(path: str):
        path = Path(path)
        if path.is_dir():
            path = path / "config.json"
        with open(path, "r", encoding="utf-8") as f:
            data = json.load(f)
        mt = data["model_type"]
        if mt == "fish_qwen3_omni":
            return BaseModelArgs._from_fish_qwen3_omni(data)
        if mt == "dual_ar":
            cls = DualARModelArgs
        elif mt == "naive":
            cls = NaiveModelArgs
        else:
            raise ValueError(f"Unknown model type: {mt}")
        valid = {f.name for f in dataclasses.fields(cls)}
        return cls(**{k: v for k, v in data.items() if k in valid})

    @staticmethod
    def _from_fish_qwen3_omni(data: dict) -> "DualARModelArgs":
        tc, adc = data["text_config"], data["audio_decoder_config"]
        flat = dict(
            model_type="dual_ar", vocab_size=tc["vocab_size"], n_layer=tc["n_layer"], n_head=tc["n_head"],
            n_local_heads=tc.get("n_local_heads", -1), head_dim=tc.get("head_dim"), dim=tc["dim"],
            intermediate_size=tc.get("intermediate_size"), rope_base=tc.get("rope_base", 10000),
            norm_eps=tc.get("norm_eps", 1e-5), max_seq_len=tc.get("max_seq_len", 2048),
            dropout=tc.get("dropout", 0.0), tie_word_embeddings=tc.get("tie_word_embeddings", True),
            attention_qkv_bias=tc.get("attention_qkv_bias", False),
            attention_o_bias=tc.get("attention_o_bias", False),
            attention_qk_norm=tc.get("attention_qk_norm", False),
            use_gradient_checkpointing=tc.get("use_gradient_checkpointing", True),
            initializer_range=tc.get("initializer_range", 0.02),
            semantic_begin_id=data.get("semantic_start_token_id", 0),
            semantic_end_id=data.get("semantic_end_token_id", 0),
            scale_codebook_embeddings=True, norm_fastlayer_input=True,
            audio_embed_dim=adc.get("text_dim", tc["dim"]), codebook_size=adc["vocab_size"],
            num_codebooks=adc["num_codebooks"], n_fast_layer=adc["n_layer"], fast_dim=adc.get("dim"),
            fast_n_head=adc.get("n_head"), fast_n_local_heads=adc.get("n_local_heads"),
            fast_head_dim=adc.get("head_dim"), fast_intermediate_size=adc.get("intermediate_size"),
            fast_attention_qkv_bias=adc.get("attention_qkv_bias"),
            fast_attention_qk_norm=adc.get("attention_qk_norm"),
            fast_attention_o_bias=adc.get("attention_o_bias"),
        )
        valid = {f.name for f in dataclasses.fields(DualARModelArgs)}
        return DualARModelArgs(**{k: v for k, v in flat.items() if k in valid and v is not None})

    def save(self, path: str):
        with open(path, "w") as f:
            json.dump(self.__dict__, f, indent=4, sort_keys=True, ensure_ascii=False)


@dataclass
class NaiveModelArgs(BaseModelArgs):
    model_type: str = "naive"


@dataclass
class DualARModelArgs(BaseModelArgs):
    model_type: str = "dual_ar"
    n_fast_layer: int = 4
    fast_dim: Optional[int] = None
    fast_n_head: Optional[int] = None
    fast_n_local_heads: Optional[int] = None
    fast_head_dim: Optional[int] = None
    fast_intermediate_size: Optional[int] = None
    fast_attention_qkv_bias: Optional[bool] = None
    fast_attention_qk_norm: Optional[bool] = None
    fast_attention_o_bias: Optional[bool] = None
    norm_fastlayer_input: bool = False

    def __post_init__(self):
        super().__post_init__()
        self.fast_dim = self.fast_dim or self.dim
        self.fast_n_head = self.fast_n_head or self.n_head
        self.fast_n_local_heads = self.fast_n_local_heads or self.n_local_heads
        self.fast_head_dim = self.fast_head_dim or self.head_dim
        self.fast_intermediate_size = self.fast_intermediate_size or self.intermediate_size
        for name, base in (("fast_attention_qkv_bias", self.attention_qkv_bias),
                           ("fast_attention_qk_norm", self.attention_qk_norm),
                           ("fast_attention_o_bias", self.attention_o_bias)):
            if getattr(self, name) is None:
                setattr(self, name, base)


def _remap_fish_qwen3_omni_keys(weights: "OrderedDict") -> "OrderedDict":
    """text_model.model.* -> *, audio_decoder.* -> fast_* (codebook_embeddings keeps its name)."""
    if not any(k.startswith(("text_model.", "audio_decoder.")) for k in weights):
        return weights
    new = OrderedDict()
    for k, v in weights.items():
        if k.startswith("text_model.model."):
            new[k[len("text_model.model."):]] = v
        elif k.startswith("audio_decoder."):
            suffix = k[len("audio_decoder."):]
            new[suffix if suffix.startswith("codebook_embeddings.") else "fast_" + suffix] = v
        else:
            new[k] = v
    return new


def _fuse_qkv(weights: dict) -> dict:
    """wq/wk/wv -> wqkv (the reference's load hook, llama.py:877-882)."""
    out = dict(weights)
    for k in list(weights):
        if k.endswith("attention.wq.weight"):
            pre = k[: -len("wq.weight")]
            out[pre + "wqkv.weight"] = torch.cat([out.pop(pre + "wq.weight"), out.pop(pre + "wk.weight"),
                                                  out.pop(pre + "wv.weight")])
    return out


class _ConfigTokenizer:
    """Fallback when no tokenizer files ship with the checkpoint: the two members the decode loop uses
    (inference.py:207, 320) served from explicit ids."""

    def __init__(self, im_end_id: int, semantic_begin_id: int):
        self._im_end_id = im_end_id
        self.semantic_begin_id = semantic_begin_id

    def get_token_id(self, token: str) -> int:
        if token != IM_END_TOKEN:
            raise KeyError(token)
        return self._im_end_id


class DualARTransformer:
    """Weights + CUDA engine behind the reference's model object surface: `.config`, `.tokenizer`,
    `.parameters()`, `.setup_caches()`, `._cache_setup_done`, `.eval()`, `.to()`."""

    def __init__(self, config: DualARModelArgs, state_dict: dict, tokenizer=None, device="cuda",
                 im_end_id: Optional[int] = None):
        self.config = config
        state_dict = _fuse_qkv(_remap_fish_qwen3_omni_keys(OrderedDict(state_dict)))
        self._state = {k: v for k, v in state_dict.items()}
        self.tokenizer = tokenizer
        if tokenizer is None:
            if im_end_id is None:
                raise ValueError("either a tokenizer or im_end_id is required")
            self.tokenizer = _ConfigTokenizer(im_end_id, config.semantic_begin_id)
        self.device = torch.device(device)
        self.dtype = torch.bfloat16
        self.engine: Optional[LmEngine] = None
        self.max_batch_size = -1
        self.max_seq_len = -1
        self.kv_pages: Optional[int] = None
        self.attn_split = 0
        self.prefix_cache = False
        self._cache_setup_done = False
        self.debug = False
        self.max_rows = 2048

    # ---- nn.Module-like surface the callers touch ----
    def parameters(self) -> Iterator[torch.Tensor]:
        if self.engine is not None:
            return iter(self.engine._keep)
        return iter(v.to(self.dtype) for v in self._state.values())

    def eval(self):
        return self

    def to(self, device=None, dtype=None):
        if dtype is not None and dtype not in (torch.bfloat16,):
            raise ValueError("fish_speech_b200 computes in bf16 (the reference's inference precision)")
        if device is not None:
            self.device = torch.device(device)
        return self

    def setup_caches(self, max_batch_size: int, max_seq_len: int, dtype: torch.dtype = torch.bfloat16,
                     kv_pages: Optional[int] = None, attn_split: int = 0, prefix_cache: bool = False):
        """llama.py:307-325 — (re)create the engine when more capacity is asked for. `kv_pages`: the slow KV
        cache's page pool (64 positions per page) when it should be smaller than every slot at full capacity.
        `attn_split`: 0 = off; else decode rows with a longer context split their attention into spans of that many
        positions (LmEngine). `prefix_cache`: prompt prefixes stay in the page pool after their slot moves on, for
        later requests to reuse (LmEngine)."""
        attn_split = int(attn_split or 0)
        prefix_cache = bool(prefix_cache)
        if (self.max_seq_len >= max_seq_len and self.max_batch_size >= max_batch_size
                and kv_pages == self.kv_pages and attn_split == self.attn_split and prefix_cache == self.prefix_cache):
            return
        max_seq_len = find_multiple(max_seq_len, 8)
        if self.engine is not None:
            self.engine.close()
        im_end = self.tokenizer.get_token_id(IM_END_TOKEN)
        self.engine = LmEngine(self.config, self._state, self.device, im_end, max_batch=max_batch_size,
                               kv_len=max_seq_len, max_rows=self.max_rows, debug=self.debug, kv_pages=kv_pages,
                               attn_split=attn_split, prefix_cache=prefix_cache)
        self.max_seq_len = max_seq_len
        self.kv_pages = kv_pages
        self.attn_split = attn_split
        self.prefix_cache = prefix_cache
        self.max_batch_size = max_batch_size

    @staticmethod
    def from_pretrained(path: str, load_weights: bool = False, max_length: Optional[int] = None,
                        lora_config=None, rope_base: Optional[int] = None, device="cuda") -> "DualARTransformer":
        """llama.py:480-594: config.json + (sharded safetensors | model.safetensors | model.pth)."""
        if lora_config is not None:
            raise NotImplementedError("LoRA is a training feature; merge it first (tools/llama/merge_lora.py)")
        config = BaseModelArgs.from_pretrained(str(path))
        if not isinstance(config, DualARModelArgs):
            raise ValueError(f"Unknown model type: {config.model_type}")
        if max_length is not None:
            config.max_seq_len = max_length
        if rope_base is not None:
            config.rope_base = rope_base
        tokenizer = None
        try:
            from fish_speech.tokenizer import FishTokenizer  # reference CPU-side tokenizer (ADJACENT)

            tokenizer = FishTokenizer.from_pretrained(path)
            # the reference injects the tokenizer's semantic id range into the config (llama.py:500-505)
            config.semantic_begin_id = tokenizer.semantic_begin_id
            config.semantic_end_id = tokenizer.semantic_end_id
        except Exception:
            tokenizer = None
        weights = OrderedDict()
        p = Path(path)
        if load_weights:
            index = p / "model.safetensors.index.json"
            single = p / "model.safetensors"
            pth = p / "model.pth"
            if index.exists():
                from safetensors.torch import load_file

                with open(index) as f:
                    shards = sorted(set(json.load(f)["weight_map"].values()))
                for s in shards:
                    weights.update(load_file(str(p / s), device="cpu"))
            elif single.exists():
                from safetensors.torch import load_file

                weights.update(load_file(str(single), device="cpu"))
            elif pth.exists():
                w = torch.load(pth, map_location="cpu", mmap=True, weights_only=True)
                if "state_dict" in w:
                    w = w["state_dict"]
                if next(iter(w.keys())).startswith("model."):
                    w = OrderedDict((k.replace("model.", ""), v) for k, v in w.items())
                weights.update((k, v) for k, v in w.items() if "audio_" not in k)
            else:
                raise FileNotFoundError(f"No model weights found in {path}")
        im_end_id = None
        if tokenizer is None:
            cfg_json = json.loads((p / "config.json").read_text()) if (p / "config.json").exists() else {}
            im_end_id = cfg_json.get("im_end_id", cfg_json.get("eos_token_id"))
        return DualARTransformer(config, weights, tokenizer=tokenizer, device=device, im_end_id=im_end_id)
