"""Drop-in surface of fish_speech/models/dac/modded_dac.py + rvq.py for inference.

`DAC` keeps the reference's public surface (`encode`, `from_indices`, `decode`, `sample_rate`, `hop_length`,
`frame_length`, `device`, `parameters()`; modded_dac.py:804-946) but holds packed device weights and
walks the reference's module tree issuing one CUDA op per layer through the C-ABI (include/fishb200.h):

  * every Conv1d / ConvTranspose1d / Linear -> fsb_conv_gemm (tcgen05 implicit-im2col GEMM, fused bias /
    Snake / GELU / LayerScale / residual epilogues); weight-norm (parametrizations.weight.original0/1) is
    folded ONCE at load instead of on every forward (modded_dac.py:554-556)
  * channels-last bf16 activations [B][T][C]; fp32 accumulation; fp32 waveform out
  * strided convs (k = m*stride) read the input as [T/stride][stride*C] rows -> m taps of K = stride*C
  * ConvTranspose1d (k = m*stride) is ONE GEMM with stride*C_out output channels and m taps
  * the window-limited transformers reuse the LM glue kernels with a banded (length-aware) attention —
    no T x T mask is ever materialised (modded_dac.py:380-398)
  * encode skips the post_module + upsample pass whose result the reference discards (rvq.py:318-319 vs
    modded_dac.py:919-923)
"""
from __future__ import annotations

import ctypes as C
import math
import threading
from dataclasses import dataclass, field
from types import MappingProxyType
from typing import Iterator, Mapping, Optional, Sequence

import torch

from ... import _lib, audio


@dataclass
class TfmConfig:
    n_layer: int = 8
    n_head: int = 16
    dim: int = 1024
    intermediate_size: int = 3072
    head_dim: int = 64
    rope_base: float = 10000
    norm_eps: float = 1e-5
    window_size: Optional[int] = 128


@dataclass
class CodecConfig:
    """Values of fish_speech/configs/modded_dac_vq.yaml (see config.load_codec_config)."""

    sample_rate: int = 44100
    encoder_dim: int = 64
    encoder_rates: tuple = (2, 4, 8, 8)
    decoder_dim: int = 1536
    decoder_rates: tuple = (8, 8, 4, 2)
    encoder_transformer_layers: tuple = (0, 0, 0, 4)
    n_codebooks: int = 9
    codebook_size: int = 1024
    semantic_codebook_size: int = 4096
    codebook_dim: int = 8
    downsample_factor: tuple = (2, 2)
    quant_tfm: TfmConfig = field(default_factory=TfmConfig)
    enc_tfm_window: int = 512

    @property
    def latent_dim(self) -> int:
        return self.encoder_dim * (2 ** len(self.encoder_rates))

    @property
    def hop_length(self) -> int:
        return int(math.prod(self.encoder_rates))

    def enc_tfm(self, dim: int, n_layer: int) -> TfmConfig:
        return TfmConfig(n_layer=n_layer, n_head=dim // 64, dim=dim, intermediate_size=dim * 3, head_dim=64,
                         rope_base=10000, norm_eps=1e-5, window_size=self.enc_tfm_window)


def _pad64(n: int) -> int:
    return (n + 63) // 64 * 64


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class _Conv:
    """A conv / linear lowered to the multi-tap GEMM: packed bf16 weight + fp32 epilogue vectors."""

    __slots__ = ("w", "bias", "c_out", "taps", "kpad", "shifts", "in_group", "out_group", "c_in_eff")

    def __init__(self, w, bias, c_out, taps, kpad, shifts, in_group=1, out_group=1, c_in_eff=0):
        self.w, self.bias, self.c_out, self.taps, self.kpad = w, bias, c_out, taps, kpad
        self.shifts = (C.c_int * len(shifts))(*shifts)
        self.in_group, self.out_group, self.c_in_eff = in_group, out_group, c_in_eff


class _Snake:
    __slots__ = ("alpha", "inv")

    def __init__(self, alpha: torch.Tensor, dev, repeat: int = 1):
        a = alpha.detach().float().reshape(-1).repeat(repeat)
        self.alpha = a.to(dev).contiguous()
        self.inv = (a + 1e-9).reciprocal().to(dev).contiguous()


class DAC:
    def __init__(self, cfg: CodecConfig, state_dict: dict, device="cuda"):
        if not torch.cuda.is_available():
            raise _lib.FsbError("fish_speech_b200 needs a CUDA device (sm_90a); there is no CPU path")
        self.lib = _lib.lib()
        self.cfg = cfg
        self._device = torch.device(device)
        self.sample_rate = cfg.sample_rate
        self.encoder_rates = list(cfg.encoder_rates)
        self.decoder_rates = list(cfg.decoder_rates)
        self.hop_length = cfg.hop_length
        self.frame_length = self.hop_length * 4  # modded_dac.py:861
        self.latent_dim = cfg.latent_dim
        self._keep: list[torch.Tensor] = []
        self._bufs: dict = {}
        self._graphs: dict = {}   # (B, S, T) -> (CUDAGraph, static index buffer, static waveform) of from_indices
        self._graph_seen: dict = {}
        self._dec_pool: Optional["DecodeStreamPool"] = None  # the streamed from_indices' pool, opened on first use
        self._ws_gen = 0  # bumped whenever a workspace or the RoPE table is re-allocated (stream pools drop their graphs)
        # decoder ResidualUnits as one kernel each (csrc/codec_resunit.cu); False = two conv GEMM launches per unit
        self._fused_units = True
        self._lock = threading.RLock()
        self._rope: dict = {}
        self._sd = {k: v.detach().float() for k, v in state_dict.items()}  # folded on the device they live on
        with torch.cuda.device(self._device):
            self._pack()
        del self._sd

    # ---- nn.Module-like surface ----
    @property
    def device(self) -> torch.device:
        return self._device

    def parameters(self) -> Iterator[torch.Tensor]:
        return iter(self._keep)

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    # -------------------------------------------------------------------------------------------
    # weight packing
    # -------------------------------------------------------------------------------------------
    def _dev(self, t: torch.Tensor, dtype) -> torch.Tensor:
        t = t.to(device=self._device, dtype=dtype).contiguous()
        self._keep.append(t)
        return t

    def _eff_weight(self, prefix: str) -> torch.Tensor:
        sd = self._sd
        g = sd.get(f"{prefix}.parametrizations.weight.original0")
        if g is None:
            return sd[f"{prefix}.weight"]
        return torch._weight_norm(sd[f"{prefix}.parametrizations.weight.original1"], g, 0)

    def _conv(self, prefix: str, dilation: int = 1, stride: int = 1) -> _Conv:
        """Conv1d weight [C_out, C_in, k] -> [C_out][taps][kpad]. stride>1 needs k % stride == 0 (the codec
        only uses k = stride and k = 2*stride)."""
        w = self._eff_weight(prefix)
        c_out, c_in, k = w.shape
        if stride == 1:
            kpad = _pad64(c_in)
            m = torch.zeros(c_out, k, kpad, device=w.device)
            m[:, :, :c_in] = w.permute(0, 2, 1)
            shifts = [-(k - 1 - j) * dilation for j in range(k)]
            taps, c_in_eff = k, c_in
        else:
            assert k % stride == 0 and dilation == 1
            taps = k // stride
            c_in_eff = stride * c_in
            kpad = _pad64(c_in_eff)
            m = torch.zeros(c_out, taps, kpad, device=w.device)
            # tap q covers kernel positions j = q*stride + r, r < stride, laid out (r, ci)
            wr = w.permute(0, 2, 1).reshape(c_out, taps, stride * c_in)
            m[:, :, :c_in_eff] = wr
            shifts = [-(taps - 1 - q) for q in range(taps)]
        bias = self._sd.get(f"{prefix}.bias")
        return _Conv(self._dev(m.reshape(c_out, taps * kpad), torch.bfloat16),
                     self._dev(bias, torch.float32) if bias is not None else None,
                     c_out, taps, kpad, shifts, in_group=stride, c_in_eff=c_in_eff)

    def _convT(self, prefix: str, stride: int) -> _Conv:
        """ConvTranspose1d weight [C_in, C_out, k], k = m*stride, right-trimmed by k - stride
        (modded_dac.py:574-580): out[t*s + p] = sum_q W[:, :, p + q*s]^T x[t - q]  -> one GEMM with
        s*C_out output channels (p major) and m taps (shift -q)."""
        w = self._eff_weight(prefix)
        c_in, c_out, k = w.shape
        assert k % stride == 0
        taps = k // stride
        kpad = _pad64(c_in)
        m = torch.zeros(stride * c_out, taps, kpad, device=w.device)
        for q in range(taps):
            # rows (p, co)  <-  W[ci, co, p + q*stride]
            blk = w[:, :, q * stride:(q + 1) * stride]  # [ci, co, p]
            m[:, q, :c_in] = blk.permute(2, 1, 0).reshape(stride * c_out, c_in)
        bias = self._sd.get(f"{prefix}.bias")
        return _Conv(self._dev(m.reshape(stride * c_out, taps * kpad), torch.bfloat16),
                     self._dev(bias.repeat(stride), torch.float32) if bias is not None else None,
                     stride * c_out, taps, kpad, [-q for q in range(taps)], out_group=stride, c_in_eff=c_in)

    def _linear(self, prefix: str, with_bias=True) -> _Conv:
        w = self._sd[f"{prefix}.weight"]
        n, k = w.shape
        kpad = _pad64(k)
        m = torch.zeros(n, kpad, device=w.device)
        m[:, :k] = w
        bias = self._sd.get(f"{prefix}.bias") if with_bias else None
        return _Conv(self._dev(m, torch.bfloat16), self._dev(bias, torch.float32) if bias is not None else None,
                     n, 1, kpad, [0], c_in_eff=k)

    def _snake(self, prefix: str, repeat: int = 1) -> _Snake:
        s = _Snake(self._sd[f"{prefix}.alpha"], self._device, repeat)
        self._keep += [s.alpha, s.inv]
        return s

    def _tfm(self, prefix: str, t: TfmConfig) -> dict:
        bf = torch.bfloat16
        layers = []
        for l in range(t.n_layer):
            p = f"{prefix}.layers.{l}"
            w13 = torch.cat([self._sd[f"{p}.feed_forward.w1.weight"], self._sd[f"{p}.feed_forward.w3.weight"]], 0)
            layers.append(dict(
                wqkv=self._dev(self._sd[f"{p}.attention.wqkv.weight"], bf),
                wo=self._dev(self._sd[f"{p}.attention.wo.weight"], bf),
                w13=self._dev(w13, bf), w2=self._dev(self._sd[f"{p}.feed_forward.w2.weight"], bf),
                attn_norm=self._dev(self._sd[f"{p}.attention_norm.weight"], bf),
                ffn_norm=self._dev(self._sd[f"{p}.ffn_norm.weight"], bf),
                ls_attn=self._dev(self._sd[f"{p}.attention_layer_scale.gamma"], bf),
                ls_ffn=self._dev(self._sd[f"{p}.ffn_layer_scale.gamma"], bf)))
        return dict(cfg=t, layers=layers, norm=self._dev(self._sd[f"{prefix}.norm.weight"], bf))

    def _convnext(self, prefix: str) -> dict:
        f32 = torch.float32
        dw = self._sd[f"{prefix}.dwconv.conv.weight"]  # [C, 1, 7]
        return dict(dw=self._dev(dw[:, 0, :], f32), dw_b=self._dev(self._sd[f"{prefix}.dwconv.conv.bias"], f32),
                    ln_w=self._dev(self._sd[f"{prefix}.norm.weight"], f32), ln_b=self._dev(self._sd[f"{prefix}.norm.bias"], f32),
                    pw1=self._linear(f"{prefix}.pwconv1"), pw2=self._linear(f"{prefix}.pwconv2"),
                    gamma=self._dev(self._sd[f"{prefix}.gamma"], f32), k=dw.shape[-1])

    def _res_unit(self, prefix: str, dilation: int) -> dict:
        return dict(s0=self._snake(f"{prefix}.block.0"), c7=self._conv(f"{prefix}.block.1.conv", dilation=dilation),
                    s1=self._snake(f"{prefix}.block.2"), c1=self._conv(f"{prefix}.block.3.conv"), dil=dilation)

    def _vq_tables(self, prefix: str):
        """out_proj(codebook) tables (fp32 [size, D]) for decode, and in_proj / normalised codebook for encode."""
        w_out = self._eff_weight(f"{prefix}.out_proj")[:, :, 0]  # [D, cd]
        cb = self._sd[f"{prefix}.codebook.weight"]  # [size, cd]
        tab = cb @ w_out.t() + self._sd[f"{prefix}.out_proj.bias"]
        w_in = self._eff_weight(f"{prefix}.in_proj")[:, :, 0]  # [cd, D]
        return tab, w_in, self._sd[f"{prefix}.in_proj.bias"], torch.nn.functional.normalize(cb)

    def _pack(self):
        cfg = self.cfg
        f32 = torch.float32
        # ---- quantizer ----
        prefixes = ["quantizer.semantic_quantizer.quantizers.0"] + [
            f"quantizer.quantizer.quantizers.{i}" for i in range(cfg.n_codebooks)]
        tabs, w_in, b_in, cbn, sizes = [], [], [], [], []
        for p in prefixes:
            tab, wi, bi, cn = self._vq_tables(p)
            tabs.append(self._dev(tab, f32))
            w_in.append(wi)
            b_in.append(bi)
            cbn.append(cn)
            sizes.append(tab.shape[0])
        self.n_stage = len(prefixes)
        self.vq_tabs = tabs
        self.vq_tab_ptrs = self._dev(torch.tensor([t.data_ptr() for t in tabs], dtype=torch.int64), torch.int64)
        self.vq_sizes = self._dev(torch.tensor(sizes, dtype=torch.int32), torch.int32)
        self.vq_in_w = self._dev(torch.stack(w_in), f32)  # [S, cd, D]
        self.vq_in_b = self._dev(torch.stack(b_in), f32)
        self.vq_cbn = self._dev(torch.cat(cbn, 0), f32)
        offs = [0]
        for s in sizes[:-1]:
            offs.append(offs[-1] + s)
        self.vq_cb_off = self._dev(torch.tensor(offs, dtype=torch.int32), torch.int32)
        self.down = [dict(conv=self._conv(f"quantizer.downsample.{i}.0.conv", stride=f),
                          cnx=self._convnext(f"quantizer.downsample.{i}.1"), f=f)
                     for i, f in enumerate(cfg.downsample_factor)]
        self.up = [dict(conv=self._convT(f"quantizer.upsample.{i}.0.conv", f),
                        cnx=self._convnext(f"quantizer.upsample.{i}.1"), f=f)
                   for i, f in enumerate(reversed(cfg.downsample_factor))]
        self.pre_tfm = self._tfm("quantizer.pre_module", cfg.quant_tfm)
        self.post_tfm = self._tfm("quantizer.post_module", cfg.quant_tfm)
        # ---- decoder ----
        self.dec_in = self._conv("decoder.model.0.conv")
        self.dec_blocks = []
        for i, s in enumerate(cfg.decoder_rates):
            p = f"decoder.model.{i + 1}.block"
            res = [self._res_unit(f"{p}.{2 + j}", d) for j, d in enumerate((1, 3, 9))]
            up_snake = _SnakeView(res[0]["s0"], s)  # Snake params in the (p, co) order of the convT GEMM
            self._keep += [up_snake.alpha, up_snake.inv]
            self.dec_blocks.append(dict(s_in=self._snake(f"{p}.0"), up=self._convT(f"{p}.1.conv", s), stride=s,
                                        res=res, up_snake=up_snake))
        n = len(cfg.decoder_rates) + 1
        self.dec_out_snake = self._snake(f"decoder.model.{n}")
        wf = self._eff_weight(f"decoder.model.{n + 1}.conv")  # [1, C, 7]
        self.dec_out_w = self._dev(wf[0].t(), f32)  # [K][C]
        self.dec_out_b = float(self._sd[f"decoder.model.{n + 1}.conv.bias"][0])
        self.dec_out_k = wf.shape[-1]
        # ---- encoder ----
        w0 = self._eff_weight("encoder.block.0.conv")  # [C0, 1, 7]
        self.enc_in_w = self._dev(w0[:, 0, :], f32)
        self.enc_in_b = self._dev(self._sd["encoder.block.0.conv.bias"], f32)
        self.enc_blocks = []
        d = cfg.encoder_dim
        for i, (s, ntl) in enumerate(zip(cfg.encoder_rates, cfg.encoder_transformer_layers)):
            d *= 2
            p = f"encoder.block.{i + 1}.block"
            self.enc_blocks.append(dict(
                res=[self._res_unit(f"{p}.{j}", dil) for j, dil in enumerate((1, 3, 9))],
                s_out=self._snake(f"{p}.3"), down=self._conv(f"{p}.4.conv", stride=s), stride=s, dim=d,
                tfm=self._tfm(f"{p}.5", cfg.enc_tfm(d, ntl)) if ntl > 0 else None))
        nb = len(cfg.encoder_rates) + 1
        self.enc_out_snake = self._snake(f"encoder.block.{nb}")
        self.enc_out = self._conv(f"encoder.block.{nb + 1}.conv")

    # -------------------------------------------------------------------------------------------
    # op helpers
    # -------------------------------------------------------------------------------------------
    def _buf(self, name: str, numel: int, dtype=torch.bfloat16) -> torch.Tensor:
        """Named persistent workspace (stable device pointers keep the GEMM plan cache small)."""
        b = self._bufs.get(name)
        if b is None or b.numel() < numel or b.dtype != dtype:
            if b is not None:
                self._graphs.clear()  # captured graphs point into the buffer that is being replaced
                self._graph_seen.clear()
                self._ws_gen += 1
            b = torch.empty(max(numel, 1), dtype=dtype, device=self._device)
            self._bufs[name] = b
        return b

    def _gemm(self, cv: _Conv, x: torch.Tensor, B: int, T_in: int, c_in: int, T_out: int, out0=None, out1=None,
              snake: Optional[_Snake] = None, resid=None, gamma=None, act=0, out_f32=False):
        """x: flat bf16 buffer viewed as [B][T_in][c_in] rows."""
        vp = lambda t: None if t is None else t.data_ptr()
        _lib.check(self.lib.fsb_conv_gemm(
            x.data_ptr(), B, T_in, c_in, c_in, T_in * c_in, cv.w.data_ptr(), cv.c_out, cv.taps, cv.kpad, cv.shifts,
            T_out, vp(cv.bias), vp(gamma), vp(resid), act, vp(out0), vp(out1),
            snake.alpha.data_ptr() if snake is not None else None,
            snake.inv.data_ptr() if snake is not None else None, int(out_f32), _stream()))

    def _rope_table(self, T: int, head_dim: int, base: float) -> torch.Tensor:
        key = (head_dim, base)
        t = self._rope.get(key)
        if t is None or t.shape[0] < T:
            n = max(T, 1024)
            inv = 1.0 / (base ** (torch.arange(0, head_dim, 2)[: head_dim // 2].float() / head_dim))
            ang = torch.outer(torch.arange(n), inv)
            cis = torch.polar(torch.ones_like(ang), ang)
            new = torch.stack([cis.real, cis.imag], dim=-1).to(torch.bfloat16).to(self._device)  # modded_dac.py:442-452
            if t is not None:
                self._graphs.clear()  # captured graphs point into the table that is being replaced
                self._graph_seen.clear()
                self._ws_gen += 1
            t = new
            self._rope[key] = t
        return t

    def _transformer(self, tf: dict, x: torch.Tensor, B: int, T: int, tag: str, pos0: int = 0,
                     kv_cache: Optional[list] = None, cache_len: int = 0, rows_at: Optional[tuple] = None,
                     ring: bool = False, rope_len: int = 0) -> torch.Tensor:
        """WindowLimitedTransformer.forward on x = flat [B*T, D] bf16 (updated in place as the residual
        stream); returns the final-normed tensor (a workspace view).
        Incremental use (DecodeStream): the T rows are positions pos0 .. pos0+T-1 of a longer sequence whose earlier
        K/V live in `kv_cache` = per layer (K, V) buffers [B][H][cache_len][Dh]; the window attention reads them.
        DecodeStreamPool: `rows_at` = (sequence, position) int32 device tensors of the B*T rows, `kv_cache` per layer
        ring buffers of `cache_len` positions (ring=True, see fsb_qkv_rope_ring), positions below `rope_len`."""
        t: TfmConfig = tf["cfg"]
        D, H, Dh, I = t.dim, t.n_head, t.head_dim, t.intermediate_size
        rows = B * T
        L = self.lib
        st = _stream()
        S = cache_len if kv_cache is not None else T
        ws = self._buf("tf_ws", rows * max(3 * H * Dh, 2 * I, D), torch.float32)
        n = self._buf("tf_n", rows * D)
        q = self._buf("tf_q", rows * H * Dh)
        kc = self._buf("tf_k", rows * H * Dh)
        vc = self._buf("tf_v", rows * H * Dh)
        att = self._buf("tf_att", rows * H * Dh)
        hb = self._buf("tf_h", rows * I)
        if rows_at is not None:
            seq, pos = rows_at
        else:
            # (sequence, position) of every row: two persistent int32 buffers refilled per call (a per-(B, T) cache
            # would grow without bound over a dataset-scale bulk encode, where almost every batch has a new shape)
            seq = self._buf("tf_seq", rows, torch.int32)[:rows]
            pos = self._buf("tf_pos", rows, torch.int32)[:rows]
            ar = torch.arange(rows, dtype=torch.int32, device=self._device)
            torch.div(ar, T, rounding_mode="floor", out=seq)
            torch.remainder(ar, T, out=pos)
            if pos0:
                pos += pos0
        freqs = self._rope_table(max(pos0 + T, rope_len), Dh, t.rope_base)
        window = t.window_size if t.window_size is not None else 0
        layers = tf["layers"]
        chk = _lib.check
        chk(L.fsb_resid_scale_norm(None, 0, None, x.data_ptr(), None, layers[0]["attn_norm"].data_ptr(), n.data_ptr(),
                                   rows, D, t.norm_eps, 0, st))
        for l, lw in enumerate(layers):
            if kv_cache is not None:
                kc, vc = kv_cache[l]
            chk(L.fsb_linear_f32(n.data_ptr(), rows, D, lw["wqkv"].data_ptr(), 3 * H * Dh, ws.data_ptr(), st))
            if ring:
                chk(L.fsb_qkv_rope_ring(ws.data_ptr(), rows, H, H, Dh, freqs.data_ptr(), seq.data_ptr(), pos.data_ptr(),
                                        q.data_ptr(), kc.data_ptr(), vc.data_ptr(), S, 1, st))
                chk(L.fsb_window_attn_ring(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), seq.data_ptr(), pos.data_ptr(),
                                           rows, H, H, Dh, S, window, 1, att.data_ptr(), st))
            else:
                chk(L.fsb_qkv_rope(ws.data_ptr(), rows, H, H, Dh, freqs.data_ptr(), seq.data_ptr(), pos.data_ptr(),
                                   q.data_ptr(), kc.data_ptr(), vc.data_ptr(), S, st))
                chk(L.fsb_window_attn(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), seq.data_ptr(), pos.data_ptr(), rows,
                                      H, H, Dh, S, window, att.data_ptr(), st))
            chk(L.fsb_linear_f32(att.data_ptr(), rows, H * Dh, lw["wo"].data_ptr(), D, ws.data_ptr(), st))
            chk(L.fsb_resid_scale_norm(ws.data_ptr(), D, lw["ls_attn"].data_ptr(), x.data_ptr(), x.data_ptr(),
                                       lw["ffn_norm"].data_ptr(), n.data_ptr(), rows, D, t.norm_eps, 0, st))
            chk(L.fsb_linear_f32(n.data_ptr(), rows, D, lw["w13"].data_ptr(), 2 * I, ws.data_ptr(), st))
            chk(L.fsb_swiglu_f32(ws.data_ptr(), rows, I, hb.data_ptr(), st))
            chk(L.fsb_linear_f32(hb.data_ptr(), rows, I, lw["w2"].data_ptr(), D, ws.data_ptr(), st))
            nxt = layers[l + 1]["attn_norm"] if l + 1 < len(layers) else tf["norm"]
            chk(L.fsb_resid_scale_norm(ws.data_ptr(), D, lw["ls_ffn"].data_ptr(), x.data_ptr(), x.data_ptr(),
                                       nxt.data_ptr(), n.data_ptr(), rows, D, t.norm_eps, 0, st))
        return n

    def _convnext_block(self, cn: dict, x: torch.Tensor, B: int, T: int, Cc: int, tag: str):
        """ConvNeXtBlock (rvq.py:173-191), in place on x (flat [B][T][C])."""
        y = self._buf("cnx_y", B * T * Cc)
        h = self._buf("cnx_h", B * T * 4 * Cc)
        _lib.check(self.lib.fsb_dwconv_ln(x.data_ptr(), cn["dw"].data_ptr(), cn["dw_b"].data_ptr(), cn["ln_w"].data_ptr(),
                                          cn["ln_b"].data_ptr(), B, T, Cc, cn["k"], 1e-6, y.data_ptr(), _stream()))
        self._gemm(cn["pw1"], y, B, T, Cc, T, out0=h, act=1)
        self._gemm(cn["pw2"], h, B, T, 4 * Cc, T, out0=x, gamma=cn["gamma"], resid=x)

    # -------------------------------------------------------------------------------------------
    # decode
    # -------------------------------------------------------------------------------------------
    # from_indices decodes through a DecodeStreamPool when the one-shot pass would not fit (see from_indices): this many
    # batch rows side by side, in pieces of this many frames (about 12 s at 44.1 kHz). Measured on an H100 (700 W,
    # tools/decode_long.py, BASELINE.md): at 5 minutes, 256-frame pieces decode one row 18 % faster than 128-frame ones
    # (0.77 GB peak), and four rows 5 % faster at 2.8 GB; 512 frames gain 9 % for one row and nothing for four, at
    # twice the memory.
    DECODE_STREAM_FRAMES = 256
    DECODE_STREAM_SLOTS = 4

    @torch.inference_mode()
    def from_indices(self, indices: torch.Tensor) -> torch.Tensor:
        """modded_dac.py:925-927: codes [B, 1+n_codebooks, T] -> waveform [B, 1, T*frame_length] (fp32).
        Like the reference (rvq.py:354-359) the caller's tensor is clamped in place.
        The ~190 launches of one decode are captured into a CUDA graph the second time a (B, T) shape is seen and
        replayed from then on: the layer walk below costs more host time than the GPU needs for short utterances.
        When the one-shot pass's workspaces fit in free device memory and its post-transformer rows (B x T) fit its
        launches (ONE_SHOT_MAX_ROWS), it runs as it always has; otherwise the batch is decoded through a
        DecodeStreamPool in pieces of DECODE_STREAM_FRAMES frames, in bounded memory and with the same samples."""
        cfg = self.cfg
        # one caller at a time per DAC object: the layers share persistent workspaces (the reference's nn.Module
        # allocates per call and may be driven from two host threads, e.g. TTSInferenceEngine + a batch encoder)
        with self._lock, torch.cuda.device(self._device):
            indices[:, 0] = torch.clamp(indices[:, 0], max=cfg.semantic_codebook_size - 1)
            indices[:, 1:] = torch.clamp(indices[:, 1:], max=cfg.codebook_size - 1)
            B, S, T = indices.shape
            key = (B, S, T)
            hit = self._graphs.get(key)
            if hit is not None:
                graph, g_idx, g_wav = hit
                g_idx.copy_(indices.reshape(-1))
                graph.replay()
                return g_wav.clone().view(B, 1, -1)
            # only a shape without a captured graph pays for the memory probe: one with a graph fit in one shot
            need = self._decode_one_shot_bytes(B, T)
            fits = need + need // 20 + self.ONE_SHOT_MARGIN_BYTES <= self._free_device_bytes()
            if not fits or B * T > self.ONE_SHOT_MAX_ROWS:
                return self._from_indices_streamed(indices)
            seen = self._graph_seen.get(key, 0)
            self._graph_seen[key] = seen + 1
            if seen == 0 or len(self._graphs) >= 4:
                # first sight of a shape (warms the plan cache and sizes the workspaces), or the graph cache is full
                idx = indices.to(device=self._device, dtype=torch.int32).contiguous()
                wav = self._from_indices_body(idx, B, S, T)
                self._idx_keepalive = idx
                return wav.view(B, 1, -1)
            g_idx = torch.empty(B * S * T, dtype=torch.int32, device=self._device)
            g_idx.copy_(indices.reshape(-1))
            torch.cuda.current_stream().synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):  # the LM worker thread keeps running
                g_wav = self._from_indices_body(g_idx.view(B, S, T), B, S, T)
            self._graphs[key] = (graph, g_idx, g_wav)
            graph.replay()
            return g_wav.clone().view(B, 1, -1)

    def _from_indices_body(self, idx: torch.Tensor, B: int, S: int, T: int) -> torch.Tensor:
        """idx int32 [B, S, T] (clamped) -> waveform [B, T*frame_length]: rvq.decode + Decoder.forward."""
        D = self.cfg.latent_dim
        z = self._buf("q_z", B * T * D)
        _lib.check(self.lib.fsb_codebook_sum(idx.data_ptr(), self.vq_tab_ptrs.data_ptr(), self.vq_sizes.data_ptr(),
                                             S, B, T, D, z.data_ptr(), _stream()))
        z = self._transformer(self.post_tfm, z, B, T, "post")
        Tc = T
        cur = z
        for i, u in enumerate(self.up):
            out = self._buf(f"up_{i}", B * Tc * u["f"] * D)
            self._gemm(u["conv"], cur, B, Tc, D, Tc, out0=out)
            Tc *= u["f"]
            self._convnext_block(u["cnx"], out, B, Tc, D, f"up{i}")
            cur = out
        return self._decoder(cur, B, Tc)

    def _decode_one_shot_bytes(self, B: int, T: int) -> int:
        """Bytes the one-shot from_indices of B x T frames would allocate: its int32 codes, the waveform and the copy a
        graph replay returns, plus every named workspace that is not already large enough (a workspace that grows is
        allocated before the old one is released). The decoder's three bf16 buffers (393 KB per frame each for the
        S2-Pro geometry) dominate."""
        cfg = self.cfg
        D, rows = cfg.latent_dim, B * T
        need = rows * self.n_stage * 4 + 2 * rows * self.frame_length * 4
        need += self._grow_bytes("q_z", rows * D) + self._tfm_bytes(self.post_tfm["cfg"], rows)
        Tc = T
        for i, f in enumerate(reversed(cfg.downsample_factor)):
            Tc *= f
            need += self._grow_bytes(f"up_{i}", B * Tc * D)
            need += self._grow_bytes("cnx_y", B * Tc * D) + self._grow_bytes("cnx_h", B * Tc * 4 * D)
        return need + sum(self._grow_bytes(f"dec_{k}", self._decoder_numel(B, Tc)) for k in range(3))

    def _from_indices_streamed(self, indices: torch.Tensor) -> torch.Tensor:
        """from_indices of clamped codes through the decode pool, row by row, into one [B, 1, T*frame_length] output."""
        B, _, T = indices.shape
        wav = torch.empty(B, 1, T * self.frame_length, dtype=torch.float32, device=self._device)
        codes = indices.to(device="cpu", dtype=torch.int32)
        self._decode_streamed(list(codes), list(wav[:, 0]))
        return wav

    @torch.inference_mode()
    def from_indices_list(self, codes: Sequence) -> list:
        """Ragged batch decode: codes of any number of utterances, each [1+n_codebooks, T_i] of any integer dtype (torch
        or numpy, T_i >= 1) -> per utterance its waveform fp32 [T_i * frame_length] on the device, in input order. Each
        equals from_indices of that utterance alone, bit for bit. The utterances share the decode pool's slots: one
        takes a slot as soon as an earlier one is done, so none is padded to a longer one beyond one push. Unlike
        from_indices, the caller's codes are not modified."""
        cfg, S = self.cfg, self.n_stage
        items = []
        for i, c in enumerate(codes):
            c = torch.as_tensor(c)
            if c.dtype.is_floating_point or c.dtype.is_complex or c.dtype == torch.bool:
                raise ValueError(f"item {i}: codes must be integers, got {c.dtype}")
            if c.ndim != 2 or c.shape[0] != S:
                raise ValueError(f"item {i}: codes must be [{S}, frames], got {tuple(c.shape)}")
            if c.shape[1] == 0:
                raise ValueError(f"item {i}: no frames")
            c = c.to(device="cpu", dtype=torch.int64)
            items.append(torch.cat([c[:1].clamp(0, cfg.semantic_codebook_size - 1),  # rvq.py:354-359, on a copy
                                    c[1:].clamp(0, cfg.codebook_size - 1)]).to(torch.int32))
        with self._lock, torch.cuda.device(self._device):
            outs = [torch.empty(c.shape[1] * self.frame_length, dtype=torch.float32, device=self._device) for c in items]
            self._decode_streamed(items, outs)
        return outs

    def _decode_streamed(self, items: list, outs: list) -> None:
        """Decode items[i] (clamped codes int32 [S, T_i] on the host) into outs[i] (fp32 [T_i * frame_length]) through
        the decode pool: up to DECODE_STREAM_SLOTS items side by side, each pushed in pieces of up to
        DECODE_STREAM_FRAMES frames; the next item takes the slot of one that is done."""
        FL, k = self.frame_length, self.DECODE_STREAM_FRAMES
        if self._dec_pool is None:  # kept: later calls replay the graphs it captured
            self._dec_pool = self.open_stream_pool(self.DECODE_STREAM_SLOTS, k_max=k)
        pool = self._dec_pool
        todo = iter(range(len(items)))
        live: dict = {}  # slot -> [item, frames decoded]
        try:
            while True:
                while len(live) < pool.slots:
                    i = next(todo, None)
                    if i is None:
                        break
                    live[pool.open()] = [i, 0]
                if not live:
                    return
                pieces = {s: items[i][:, f: f + k] for s, (i, f) in live.items()}
                for s, wav in pool.push(pieces).items():
                    i, f = live[s]
                    n = pieces[s].shape[1]
                    outs[i][f * FL: (f + n) * FL].copy_(wav)
                    if f + n == items[i].shape[1]:
                        pool.close(s)
                        del live[s]
                    else:
                        live[s][1] = f + n
        finally:
            for s in live:
                pool.close(s)

    def open_decode_stream(self, batch: int = 1, max_frames: int = 4096, conv_context: int = 16,
                           sample_rate: Optional[int] = None, sample_format: Optional[str] = None) -> "DecodeStream":
        """Incremental `from_indices` (SURVEY §8(f).3): push code frames as the LM emits them, get their samples back.
        The codec is causal (rvq.py:395-398 asserts it), so what a frame sounds like never depends on later frames.
        With a `sample_rate` or `sample_format` (see audio.convert_out) the samples come converted, and `flush()` at
        the end returns the ones the resampler's look-ahead held back."""
        return DecodeStream(self, batch, max_frames, conv_context, sample_rate, sample_format)

    def open_stream_pool(self, slots: int, k_max: int = 32, max_graphs: int = 8) -> "DecodeStreamPool":
        """Streaming decode of up to `slots` independent streams at once: streams join and leave at any push, and one
        push decodes the new frames of every stream that has some in one batched (graph-replayed) pass. Each stream's
        audio is bit-identical to `from_indices` of its codes alone. See DecodeStreamPool."""
        return DecodeStreamPool(self, slots, k_max, max_graphs)

    @torch.inference_mode()
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """modded_dac.py:929-946: latent [B, D, T'] (channels first) -> waveform [B, 1, T'*hop]."""
        with self._lock, torch.cuda.device(self._device):
            B, D, Tc = z.shape
            buf = self._buf("dec_zin", B * Tc * D)
            buf[: B * Tc * D].view(B, Tc, D).copy_(z.to(self._device).transpose(1, 2))
            return self._decoder(buf, B, Tc).view(B, 1, -1)

    def _unit_is_fusable(self, ru: dict, c: int) -> bool:
        c7, c1 = ru["c7"], ru["c1"]
        return (self._fused_units and c7.taps == 7 and c1.taps == 1 and c7.bias is not None and c1.bias is not None
                and c7.kpad == _pad64(c) and c1.kpad == _pad64(c) and bool(self.lib.fsb_res_unit_supported(c)))

    def _decoder_numel(self, B: int, T: int) -> int:
        """Elements of each of the decoder's buffers for B x T latent rows: its largest activation."""
        cfg = self.cfg
        numel = max(B * (T * math.prod(cfg.decoder_rates[: i + 1])) * (cfg.decoder_dim // 2 ** (i + 1))
                    for i in range(len(cfg.decoder_rates)))
        return max(numel, B * T * cfg.decoder_dim)

    def _decoder(self, z: torch.Tensor, B: int, T: int) -> torch.Tensor:
        """Decoder.forward (modded_dac.py:760-801) on z = flat [B][T][latent] bf16."""
        cfg = self.cfg
        c = cfg.decoder_dim
        t_full = T * cfg.hop_length
        bufs = [self._buf(f"dec_{k}", self._decoder_numel(B, T)) for k in range(3)]
        free = [0, 1, 2]

        def take():
            return free.pop(0)

        a = take()
        first = self.dec_blocks[0]
        self._gemm(self.dec_in, z, B, T, cfg.latent_dim, T, out1=bufs[a], snake=first["s_in"])
        Tc, cin = T, c
        for bi, blk in enumerate(self.dec_blocks):
            s = blk["stride"]
            cout = cin // 2
            x, a2 = take(), take()
            # transposed conv: raw -> x (residual stream), Snake(res0.block.0) -> a2
            self._gemm(blk["up"], bufs[a], B, Tc, cin, Tc, out0=bufs[x], out1=bufs[a2], snake=blk["up_snake"])
            free.append(a)
            Tc *= s
            a = a2
            for j, ru in enumerate(blk["res"]):
                m = take()
                last_unit = j == 2
                if not last_unit:
                    nxt = blk["res"][j + 1]["s0"]
                elif bi + 1 < len(self.dec_blocks):
                    nxt = self.dec_blocks[bi + 1]["s_in"]
                else:
                    nxt = self.dec_out_snake
                keep_raw = not last_unit
                if self._unit_is_fusable(ru, cout):
                    # Snake -> conv7 -> Snake -> conv1 -> + x in one kernel; the activated result goes to the spare buffer
                    # (neighbouring tiles still read their halo from bufs[a])
                    c7, c1 = ru["c7"], ru["c1"]
                    _lib.check(self.lib.fsb_res_unit(
                        bufs[a].data_ptr(), bufs[x].data_ptr(), B, Tc, cout, ru["dil"], c7.w.data_ptr(), c7.bias.data_ptr(),
                        ru["s1"].alpha.data_ptr(), ru["s1"].inv.data_ptr(), c1.w.data_ptr(), c1.bias.data_ptr(),
                        bufs[x].data_ptr() if keep_raw else None, bufs[m].data_ptr(), nxt.alpha.data_ptr(),
                        nxt.inv.data_ptr(), _stream()))
                    free.append(a)
                    a = m
                    continue
                self._gemm(ru["c7"], bufs[a], B, Tc, cout, Tc, out1=bufs[m], snake=ru["s1"])
                self._gemm(ru["c1"], bufs[m], B, Tc, cout, Tc, out0=bufs[x] if keep_raw else None, out1=bufs[a],
                           snake=nxt, resid=bufs[x])
                free.append(m)
            free.append(x)
            cin = cout
        wav = torch.empty(B, t_full, dtype=torch.float32, device=self._device)
        _lib.check(self.lib.fsb_final_conv_tanh(bufs[a].data_ptr(), self.dec_out_w.data_ptr(), self.dec_out_b, B, Tc, cin,
                                                self.dec_out_k, wav.data_ptr(), _stream()))
        return wav

    # -------------------------------------------------------------------------------------------
    # encode
    # -------------------------------------------------------------------------------------------
    # encode and from_indices route to the streamed path when their one-shot workspaces would not fit in free device
    # memory with a margin of this plus 5 % of the estimate left over (the caching allocator's rounding, the small
    # buffers the estimate omits)
    ONE_SHOT_MARGIN_BYTES = 512 << 20
    # the transformers' row-wise glue kernels launch one CTA row per token row (grid.y), so one pass takes at most this
    # many rows per transformer: for the S2-Pro encoder transformer (4 rows per frame) about 12.7 minutes of audio, for
    # the post-transformer of from_indices (1 row per frame) about 50 minutes
    ONE_SHOT_MAX_ROWS = 65535
    ENCODE_STREAM_FRAMES = 128  # frames per push of the streamed path (about 6 s at 44.1 kHz)
    ENCODE_STREAM_SLOTS = 4  # batch rows encoded side by side by the streamed path

    @torch.inference_mode()
    def encode(self, audio_data: torch.Tensor, audio_lengths: Optional[torch.Tensor] = None,
               n_quantizers: Optional[int] = None, **kwargs):
        """modded_dac.py:874-923: audio [B,1,N] or [B,N] -> (codes int64 [B, 1+n_codebooks, T], lens [B]).
        When the one-shot pass's workspaces fit in free device memory and its transformer rows fit its launches
        (ONE_SHOT_MAX_ROWS), it runs as it always has; otherwise the batch is encoded through an EncodeStreamPool in
        pieces of ENCODE_STREAM_FRAMES frames, in bounded memory and with the same codes and lengths."""
        with self._lock, torch.cuda.device(self._device):
            B, length = audio_data.shape[0], audio_data.shape[-1]
            N = math.ceil(length / self.frame_length) * self.frame_length
            need = self._encode_one_shot_bytes(B, N)
            rows = max(r for _, r in self._encode_one_shot_tfm_rows(B, N))
            fits = need + need // 20 + self.ONE_SHOT_MARGIN_BYTES <= self._free_device_bytes()
            if fits and rows <= self.ONE_SHOT_MAX_ROWS:
                return self._encode_one_shot(audio_data, audio_lengths, n_quantizers)
            return self._encode_streamed(audio_data, audio_lengths, n_quantizers)

    def _free_device_bytes(self) -> int:
        """Device memory a new allocation can use: free on the device plus what the caching allocator holds unused."""
        free, _ = torch.cuda.mem_get_info(self._device)
        return free + torch.cuda.memory_reserved(self._device) - torch.cuda.memory_allocated(self._device)

    def _encode_one_shot_bytes(self, B: int, N: int) -> int:
        """Bytes the one-shot encode of B x N padded samples would allocate: its fp32 waveform copy and codes, plus every
        named workspace that is not already large enough (a workspace that grows is allocated before the old one is
        released). The bf16 encoder activations (3 x B x N x encoder_dim) dominate."""
        cfg = self.cfg
        grow = self._grow_bytes
        need = 2 * B * N * 4  # the padded fp32 waveform (and the input's conversion to it)
        need += sum(grow(f"enc_{k}", B * N * cfg.encoder_dim) for k in range(3))
        T = N // self.hop_length
        D = cfg.latent_dim
        need += grow("enc_z", B * T * D)
        for i, f in enumerate(cfg.downsample_factor):
            T //= f
            need += grow(f"down_{i}", B * T * D) + grow("cnx_y", B * T * D) + grow("cnx_h", B * T * 4 * D)
        for tf, rows in self._encode_one_shot_tfm_rows(B, N):
            need += self._tfm_bytes(tf["cfg"], rows)
        need += B * self.n_stage * T * (4 + 8)  # int32 codes and their int64 copy
        return need

    def _grow_bytes(self, name: str, numel: int, elt: int = 2, dtype=torch.bfloat16) -> int:
        """Bytes `_buf(name, numel, dtype)` would allocate: 0 when the workspace is already large enough."""
        b = self._bufs.get(name)
        return 0 if b is not None and b.numel() >= numel and b.dtype == dtype else max(numel, 1) * elt

    def _tfm_bytes(self, t: TfmConfig, rows: int) -> int:
        """Bytes the workspaces of `_transformer` over `rows` rows would allocate."""
        grow, HD = self._grow_bytes, t.n_head * t.head_dim
        need = grow("tf_ws", rows * max(3 * HD, 2 * t.intermediate_size, t.dim), 4, torch.float32)
        need += grow("tf_n", rows * t.dim) + sum(grow(f"tf_{k}", rows * HD) for k in ("q", "k", "v", "att"))
        return need + grow("tf_h", rows * t.intermediate_size) + 3 * rows * 4  # + row (sequence, position), arange

    def _encode_one_shot_tfm_rows(self, B: int, N: int) -> list:
        """(transformer, rows) of every transformer the one-shot encode of B x N padded samples runs."""
        out = [(blk["tfm"], B * N // math.prod(self.encoder_rates[: i + 1]))
               for i, blk in enumerate(self.enc_blocks) if blk["tfm"] is not None]
        return out + [(self.pre_tfm, B * N // self.hop_length // math.prod(self.cfg.downsample_factor))]

    def _encode_streamed(self, audio_data: torch.Tensor, audio_lengths: Optional[torch.Tensor],
                         n_quantizers: Optional[int]):
        """encode through an EncodeStreamPool: ENCODE_STREAM_SLOTS batch rows at a time, each pushed as whole frames of
        its waveform zero-padded to the batch's padded length, as the one-shot pass sees it."""
        FL = self.frame_length
        B, length = audio_data.shape[0], audio_data.shape[-1]
        wav = audio_data.reshape(B, length)
        T = math.ceil(length / FL)
        k = self.ENCODE_STREAM_FRAMES
        pool = self.open_encode_pool(min(B, self.ENCODE_STREAM_SLOTS), k_max=k, n_quantizers=n_quantizers)
        codes = torch.empty(B, pool.n_stage, T, dtype=torch.int64, device=self._device)
        for b0 in range(0, B, pool.slots):
            rows = range(b0, min(B, b0 + pool.slots))
            slot = {b: pool.open() for b in rows}
            for f0 in range(0, T, k):
                f1 = min(T, f0 + k)
                pieces = {}
                for b in rows:
                    piece = wav[b, f0 * FL: f1 * FL].to(torch.float32)
                    if piece.numel() < (f1 - f0) * FL:  # encode's right pad
                        piece = torch.nn.functional.pad(piece, (0, (f1 - f0) * FL - piece.numel()))
                    pieces[slot[b]] = piece
                out = pool.push(pieces)
                for b in rows:
                    codes[b, :, f0:f1] = out[slot[b]]
            for b in rows:
                pool.close(slot[b])
        if audio_lengths is None:
            audio_lengths = torch.LongTensor([T * FL])
        indices_lens = torch.ceil(audio_lengths.to(self._device) / FL).long()
        return codes, indices_lens

    def open_encode_pool(self, slots: int, k_max: int = 32, n_quantizers: Optional[int] = None,
                         max_graphs: int = 8) -> "EncodeStreamPool":
        """Streaming `encode` of up to `slots` independent streams at once: streams join and leave at any push, and one
        push encodes the new frames of every stream that has some in one batched (graph-replayed) pass, in memory that
        does not grow with a stream's length. Each stream's codes are bit-identical to `encode` of its waveform alone.
        A stream opened with `open(sample_rate=sr)` takes audio at `sr` in pieces of any length and ends with `flush`.
        See EncodeStreamPool."""
        return EncodeStreamPool(self, slots, k_max, n_quantizers, max_graphs)

    def _encode_one_shot(self, audio_data: torch.Tensor, audio_lengths: Optional[torch.Tensor],
                         n_quantizers: Optional[int]):
        """Every layer over the whole (padded) batch at once."""
        cfg = self.cfg
        if audio_data.ndim == 2:
            audio_data = audio_data.unsqueeze(1)
        length = audio_data.shape[-1]
        right_pad = math.ceil(length / self.frame_length) * self.frame_length - length
        wav = torch.nn.functional.pad(audio_data.to(device=self._device, dtype=torch.float32), (0, right_pad))
        if audio_lengths is None:
            audio_lengths = torch.LongTensor([length + right_pad]).to(self._device)
        B, _, N = wav.shape
        wav = wav.reshape(B, N).contiguous()
        d0 = cfg.encoder_dim
        numel = B * N * d0
        bufs = [self._buf(f"enc_{k}", numel) for k in range(3)]
        x, a, m = 0, 1, 2
        r0 = self.enc_blocks[0]["res"][0]
        _lib.check(self.lib.fsb_first_conv(wav.data_ptr(), self.enc_in_w.data_ptr(), self.enc_in_b.data_ptr(),
                                           r0["s0"].alpha.data_ptr(), r0["s0"].inv.data_ptr(), B, N, d0,
                                           self.enc_in_w.shape[1], bufs[x].data_ptr(), bufs[a].data_ptr(), _stream()))
        Tc, c = N, d0
        for bi, blk in enumerate(self.enc_blocks):
            for j, ru in enumerate(blk["res"]):
                self._gemm(ru["c7"], bufs[a], B, Tc, c, Tc, out1=bufs[m], snake=ru["s1"])
                nxt = blk["res"][j + 1]["s0"] if j < 2 else blk["s_out"]
                self._gemm(ru["c1"], bufs[m], B, Tc, c, Tc, out0=bufs[x] if j < 2 else None, out1=bufs[a],
                           snake=nxt, resid=bufs[x])
            s, cout = blk["stride"], blk["dim"]
            Tn = Tc // s
            # strided conv reads the activation as [Tc/s][s*c] rows
            last = bi + 1 == len(self.enc_blocks)
            if blk["tfm"] is not None:
                self._gemm(blk["down"], bufs[a], B, Tn, s * c, Tn, out0=bufs[x])
                n_out = self._transformer(blk["tfm"], bufs[x], B, Tn, f"enc{bi}")
                sn = self.enc_out_snake if last else self.enc_blocks[bi + 1]["res"][0]["s0"]
                _lib.check(self.lib.fsb_snake(n_out.data_ptr(), sn.alpha.data_ptr(), sn.inv.data_ptr(),
                                              B * Tn * cout, cout, bufs[a].data_ptr(), _stream()))
                bufs[x][: B * Tn * cout].copy_(n_out[: B * Tn * cout])
            else:
                sn = self.enc_out_snake if last else self.enc_blocks[bi + 1]["res"][0]["s0"]
                self._gemm(blk["down"], bufs[a], B, Tn, s * c, Tn, out0=bufs[x], out1=bufs[m], snake=sn)
                a, m = m, a
            Tc, c = Tn, cout
        z = self._buf("enc_z", B * Tc * cfg.latent_dim)
        self._gemm(self.enc_out, bufs[a], B, Tc, c, Tc, out0=z)
        # ---- quantizer.forward up to the codes (rvq.py:293-317) ----
        D = cfg.latent_dim
        cur = z
        for i, dn in enumerate(self.down):
            f = dn["f"]
            Tn = Tc // f
            out = self._buf(f"down_{i}", B * Tn * D)
            self._gemm(dn["conv"], cur, B, Tn, f * D, Tn, out0=out)
            self._convnext_block(dn["cnx"], out, B, Tn, D, f"down{i}")
            cur, Tc = out, Tn
        zq = self._transformer(self.pre_tfm, cur, B, Tc, "pre")
        S = self.n_stage if n_quantizers is None else min(self.n_stage, 1 + int(n_quantizers))
        codes = torch.empty(B, S, Tc, dtype=torch.int32, device=self._device)
        _lib.check(self.lib.fsb_vq_encode(zq.data_ptr(), self.vq_in_w.data_ptr(), self.vq_in_b.data_ptr(),
                                          self.vq_cbn.data_ptr(), self.vq_cb_off.data_ptr(), self.vq_sizes.data_ptr(),
                                          self.vq_tab_ptrs.data_ptr(), S, cfg.codebook_dim, B, Tc, D,
                                          codes.data_ptr(), _stream()))
        indices_lens = torch.ceil(audio_lengths.to(self._device) / self.frame_length).long()
        return codes.long(), indices_lens


class DecodeStream:
    """Streaming state of one `from_indices` over a growing code sequence (one per utterance batch).

    * post-transformer (8 layers, causal window 128): K/V of every layer stay in a cache; a push computes only the new
      frames at their absolute positions (the kernels are the ones the whole-sequence path uses: row positions + cache
      length are arguments) -- exact.
    * upsample + decoder convolutions: causal with a finite receptive field (< 10 frames: dilated k7 convs at 4..512
      steps per frame, ConvNeXt k7 at 2 and 4 steps per frame); the last `conv_context` frames of the transformer
      OUTPUT are kept and re-run in front of the new frames, and only the new frames' samples are returned -- exact
      as long as conv_context covers the receptive field (tests compare with the one-shot decode).
    """

    def __init__(self, dac: "DAC", batch: int, max_frames: int, conv_context: int,
                 sample_rate: Optional[int] = None, sample_format: Optional[str] = None):
        self.dac, self.B, self.S, self.ctx = dac, int(batch), int(max_frames), int(conv_context)
        # one output converter per row, when a rate or format is asked for
        self.out = None if sample_rate is None and sample_format is None else [
            audio.OutputStream(sample_rate, sample_format, dac.device, orig_freq=dac.sample_rate)
            for _ in range(self.B)]
        t: TfmConfig = dac.post_tfm["cfg"]
        dev = dac.device
        n = self.B * t.n_head * self.S * t.head_dim
        self.kv = [(torch.zeros(n, dtype=torch.bfloat16, device=dev), torch.zeros(n, dtype=torch.bfloat16, device=dev))
                   for _ in dac.post_tfm["layers"]]
        self.pos = 0
        self.tail: Optional[torch.Tensor] = None  # [B, <=ctx, D] transformer output of the latest frames

    @torch.inference_mode()
    def push(self, indices: torch.Tensor) -> torch.Tensor:
        """codes [B, 1+n_codebooks, k] of the next k frames -> waveform [B, 1, k * frame_length] (fp32), or with a
        rate or format the samples of each row converted so far [B, 1, m]."""
        wav = self._push(indices)
        return wav if self.out is None else self._convert([w for w in wav[:, 0]])

    @torch.inference_mode()
    def flush(self) -> torch.Tensor:
        """End of the stream: [B, 1, m], the converted samples pushes held back ([B, 1, 0] fp32 without conversion)."""
        if self.out is None:
            return torch.zeros(self.B, 1, 0, dtype=torch.float32, device=self.dac.device)
        return self._convert([None] * self.B)

    def _convert(self, pieces: list) -> torch.Tensor:
        with self.dac._lock, torch.cuda.device(self.dac.device):
            ys = audio.OutputStream.push_many(list(zip(self.out, pieces)))
        return torch.stack(ys)[:, None]

    def _push(self, indices: torch.Tensor) -> torch.Tensor:
        dac, cfg = self.dac, self.dac.cfg
        B, S_, k = indices.shape
        if B != self.B:
            raise ValueError(f"stream was opened for batch {self.B}, got {B}")
        if self.out is not None and self.out[0].counts.done:
            raise ValueError("the stream was flushed")
        if k == 0:
            return torch.zeros(B, 1, 0, dtype=torch.float32, device=dac.device)
        if self.pos + k > self.S:
            raise ValueError(f"decode stream capacity exceeded ({self.pos} + {k} > {self.S} frames)")
        with dac._lock, torch.cuda.device(dac.device):
            idx = indices.to(device=dac.device, dtype=torch.int32).clone()
            idx[:, 0].clamp_(max=cfg.semantic_codebook_size - 1)  # rvq.py:354-359
            idx[:, 1:].clamp_(max=cfg.codebook_size - 1)
            idx = idx.contiguous()
            D = cfg.latent_dim
            z = dac._buf("st_z", B * k * D)
            _lib.check(dac.lib.fsb_codebook_sum(idx.data_ptr(), dac.vq_tab_ptrs.data_ptr(), dac.vq_sizes.data_ptr(), S_, B,
                                                k, D, z.data_ptr(), _stream()))
            zn = dac._transformer(dac.post_tfm, z, B, k, "post", pos0=self.pos, kv_cache=self.kv, cache_len=self.S)
            new = zn[: B * k * D].view(B, k, D)
            seq = new if self.tail is None else torch.cat([self.tail, new], dim=1)
            c = seq.shape[1] - k  # context frames in front of the new ones
            Tc = seq.shape[1]
            cur = dac._buf("st_in", B * Tc * D)
            cur[: B * Tc * D].view(B, Tc, D).copy_(seq)
            for i, u in enumerate(dac.up):
                out = dac._buf(f"up_{i}", B * Tc * u["f"] * D)
                dac._gemm(u["conv"], cur, B, Tc, D, Tc, out0=out)
                Tc *= u["f"]
                dac._convnext_block(u["cnx"], out, B, Tc, D, f"up{i}")
                cur = out
            wav = dac._decoder(cur, B, Tc).view(B, 1, -1)
            self.tail = seq[:, -self.ctx:].clone() if self.ctx > 0 else None
            self.pos += k
            dac._idx_keepalive = idx
            return wav[:, :, c * dac.frame_length:]


def _pow2(n: int) -> int:
    return 1 << max(0, int(n) - 1).bit_length()


class _StreamPool:
    """Slot, bucket and CUDA-graph bookkeeping shared by DecodeStreamPool and EncodeStreamPool.

    A subclass sets `layers` (one (history rows, row width in bf16 units, rows per frame) per windowed conv input, in
    execution order), `kv` (its transformers' ring K/V) and `_tfms` ((TfmConfig, rows per frame) per transformer), and
    supplies the piece-specific parts of a push: `_check_piece`, `_frames`, `_describe` (host-side description of a
    push), `_alloc_static` / `_stage` (the device buffers a pass reads), `_body` (the device work) and `_outputs`."""

    _fill = "fsb_window_fill"  # the entry point that builds a layer's input window

    def __init__(self, dac: "DAC", slots: int, k_max: int, max_graphs: int):
        self.dac, self.slots, self.k_max, self.max_graphs = dac, int(slots), int(k_max), int(max_graphs)
        self.hist = [torch.zeros(max(1, self.slots * H * Cc), dtype=torch.bfloat16, device=dac.device)
                     for H, Cc, _ in self.layers]
        self.rates = sorted({r for _, _, r in self.layers})
        self.pos = [0] * self.slots
        self.live = [False] * self.slots
        self.broken = [False] * self.slots
        self._graphs: dict = {}  # (nb, kb) -> (CUDAGraph, static result)
        self._seen: dict = {}
        self._gen = dac._ws_gen
        self._static: dict = {}  # (nb, kb) -> device buffers the pass reads
        self._shifts: dict = {}

    @property
    def state_bytes(self) -> int:
        """Device memory of the per-slot state (K/V rings and per-layer conv history)."""
        return sum(t.numel() * t.element_size() for kv in self.kv for t in kv) + \
            sum(h.numel() * h.element_size() for h in self.hist)

    def open(self) -> int:
        with self.dac._lock, torch.cuda.device(self.dac.device):
            for s in range(self.slots):
                if not self.live[s]:
                    for (H, Cc, _), h in zip(self.layers, self.hist):
                        if H:
                            h[s * H * Cc: (s + 1) * H * Cc].zero_()  # zero history = the one-shot's zero fill
                    self.live[s], self.broken[s], self.pos[s] = True, False, 0
                    return s
        raise ValueError(f"stream pool is full ({self.slots} slots)")

    def close(self, slot: int) -> None:
        with self.dac._lock:
            self._check_slot(slot)
            self.live[slot] = False

    def n_open(self) -> int:
        return sum(self.live)

    def _check_slot(self, slot) -> None:
        if not isinstance(slot, int) or not 0 <= slot < self.slots or not self.live[slot]:
            raise ValueError(f"slot {slot!r} is not an open stream of this pool")

    @torch.inference_mode()
    def push(self, pieces: dict) -> dict:
        """{slot: next piece of that stream} -> {slot: its result} (the piece and result formats are the subclass's).
        The caller's tensors are not modified."""
        dac = self.dac
        items = list(pieces.items())
        for slot, piece in items:
            self._check_slot(slot)
            if self.broken[slot]:
                raise ValueError(f"slot {slot}: an earlier push failed, its state is lost; close the slot")
            self._check_piece(slot, piece)
        if not items:
            return {}
        ks = [self._frames(piece) for _, piece in items]
        nb = min(_pow2(len(items)), self.slots)
        kb = min(_pow2(max(ks)), self.k_max)
        with dac._lock, torch.cuda.device(dac.device):
            host = self._describe(items, ks, nb, kb)
            # ---- the RoPE table must cover every position before a graph captures its address ----
            top = max(self.pos[s] + k for (s, _), k in zip(items, ks))
            rope_len = max(1024, _pow2(max(top, kb) * max(r for _, r in self._tfms)))
            for t, _ in self._tfms:
                dac._rope_table(rope_len, t.head_dim, t.rope_base)
            if self._gen != dac._ws_gen:  # a workspace a graph points into was re-allocated
                self._graphs.clear()
                self._seen.clear()
                self._gen = dac._ws_gen
            key = (nb, kb)
            st = self._static.get(key)
            if st is None:
                st = self._alloc_static(nb, kb, host)
                self._static[key] = st
            try:
                self._stage(st, items, ks, host)
                hit = self._graphs.get(key)
                if hit is not None:
                    hit[0].replay()
                    res = hit[1]
                else:
                    seen = self._seen.get(key, 0)
                    self._seen[key] = seen + 1
                    if seen == 0 or len(self._graphs) >= self.max_graphs:
                        res = self._body(nb, kb, st, rope_len)
                    else:
                        torch.cuda.current_stream().synchronize()
                        graph = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(graph, capture_error_mode="thread_local"):  # other threads keep running
                            res = self._body(nb, kb, st, rope_len)
                        if self._gen != dac._ws_gen:
                            raise RuntimeError("stream pool: a workspace was re-allocated during graph capture")
                        self._graphs[key] = (graph, res)
                        graph.replay()
                out = self._outputs(res, items, ks)
            except BaseException:
                for slot, _ in items:  # the device work may have advanced part of their state
                    self.broken[slot] = True
                raise
            for slot, k in zip(pieces, ks):
                self.pos[slot] += k
            return out

    def _gemm_win(self, cv: _Conv, win: torch.Tensor, nb: int, H: int, n: int, c_in: int, out0=None, out1=None,
                  snake: Optional[_Snake] = None, resid=None):
        """Conv GEMM over a window [nb][H + n][c_in]: only the n new rows, taps shifted by the H history rows."""
        sh = self._shifts.get((id(cv), H))
        if sh is None:
            sh = (C.c_int * cv.taps)(*[v + H for v in cv.shifts])
            self._shifts[(id(cv), H)] = sh
        vp = lambda t: None if t is None else t.data_ptr()
        _lib.check(self.dac.lib.fsb_conv_gemm(
            win.data_ptr(), nb, H + n, c_in, c_in, (H + n) * c_in, cv.w.data_ptr(), cv.c_out, cv.taps, cv.kpad, sh, n,
            vp(cv.bias), None, vp(resid), 0, vp(out0), vp(out1),
            snake.alpha.data_ptr() if snake is not None else None,
            snake.inv.data_ptr() if snake is not None else None, 0, _stream()))

    def _windows(self, nb: int, slot_t: torch.Tensor, valid: dict, ws: str):
        """A function (dense new rows [nb][n][row], n) -> (window of the next windowed layer, its history rows H): fills
        the window from the slot's history and the new rows and rolls the slot's history (layers in execution order)."""
        dac, L, chk = self.dac, self.dac.lib, _lib.check
        fill = getattr(L, self._fill)
        layer = iter(range(len(self.layers)))

        def window(dense: torch.Tensor, n: int):
            li = next(layer)
            H, Cc, r = self.layers[li]
            win = dac._buf(ws, nb * (H + n) * Cc)
            chk(fill(self.hist[li].data_ptr(), dense.data_ptr(), win.data_ptr(), slot_t.data_ptr(), valid[r].data_ptr(),
                     nb, H, n, Cc * 2, _stream()))
            chk(L.fsb_window_roll(win.data_ptr(), self.hist[li].data_ptr(), slot_t.data_ptr(), valid[r].data_ptr(),
                                  nb, H, n, Cc * 2, _stream()))
            return win, H

        return window


class DecodeStreamPool(_StreamPool):
    """Streaming `from_indices` of up to `slots` independent streams (one utterance each), decoded together; a push
    computes only the new frames of the streams in it: push({slot: codes [1+n_codebooks, k]}, 1 <= k <= k_max) ->
    {slot: waveform fp32 [k * frame_length]}.

    * post-transformer: per slot and layer a K/V ring of R = round_up(window + k_max + 63, 64) positions
      (fsb_qkv_rope_ring / fsb_window_attn_ring): the attention walks the same absolute 64-position tiles as over a
      linear cache, so the result is the same; memory is fixed per slot and a stream has no length cap.
    * upsampler + decoder: every causal conv keeps its own left context per slot, the last (taps - 1) * dilation rows
      of its input in the form the conv reads it (Snake-activated where the Snake is fused upstream): ConvTranspose 1
      row, ConvNeXt depthwise 6, the dilated k7 convs 6 * d, the final conv K - 1. A layer's input is a window
      [stream][H + new rows][C]: fsb_window_fill puts the slot's history in rows 0..H-1 and the producer's new rows after
      it, the consumer computes only the new rows (conv GEMM taps shifted by H, fsb_dwconv_ln_window), and
      fsb_window_roll keeps the last H valid rows as the slot's next history. At stream start the history is zeros, as
      the zero fill at negative time of the one-shot decode. The decoder's ResidualUnits run as their two conv GEMMs
      (bit-identical to the fused kernel); the final conv runs over the window and its history rows are dropped.
    * ragged pushes: the streams are padded to the largest frame count; padding rows follow a stream's valid rows, so
      a causal layer never carries them into a valid row, and the roll takes valid rows only. Padding rows of the
      transformer attend in a scratch sequence of their own. Slots outside a push are not touched.
    * each (stream bucket, frame bucket) shape, powers of two, is captured into a CUDA graph the second time it is seen
      (at most `max_graphs`; others run eagerly), on the calling thread.
    * a push that fails leaves the state of its slots undefined: they refuse further pushes until closed.
    """

    def __init__(self, dac: "DAC", slots: int, k_max: int, max_graphs: int):
        t: TfmConfig = dac.post_tfm["cfg"]
        if slots < 1 or k_max < 1:
            raise ValueError(f"stream pool needs slots >= 1 and k_max >= 1 (got {slots}, {k_max})")
        if not t.window_size or t.window_size <= 0:
            raise ValueError("stream pool needs a window-limited post-transformer")
        self.dac = dac
        self.ring = _pad64(t.window_size + int(k_max) + 63)
        # slot `slots` is the scratch sequence of padding rows
        n = (int(slots) + 1) * t.n_head * (self.ring + 64) * t.head_dim
        self.kv = [(torch.zeros(n, dtype=torch.bfloat16, device=dac.device),
                    torch.zeros(n, dtype=torch.bfloat16, device=dac.device)) for _ in dac.post_tfm["layers"]]
        self._tfms = [(t, 1)]
        # one (H rows, C channels, rows per frame) per conv input of the upsampler + decoder, in execution order
        self.layers = self._layer_geometry()
        self._out: dict = {}  # slot -> audio.OutputStream, for slots opened with a sample rate or format
        super().__init__(dac, slots, k_max, max_graphs)

    def open(self, sample_rate: Optional[int] = None, sample_format: Optional[str] = None) -> int:
        """A new stream's slot. Without a rate or format its pushes return fp32 at the codec's rate, as always; with
        either, they return the samples converted so far (audio.OutputStream: torchaudio's resampler, then float32,
        pcm16 = int16 or mulaw = uint8), and `flush(slot)` returns the rest."""
        conv = sample_rate is not None or sample_format is not None
        if conv:  # check the arguments before a slot is taken
            out = audio.OutputStream(sample_rate, sample_format, self.dac.device, orig_freq=self.dac.sample_rate)
        with self.dac._lock, torch.cuda.device(self.dac.device):
            slot = super().open()
            if conv:
                self._out[slot] = out
            return slot

    def close(self, slot: int) -> None:
        with self.dac._lock:
            super().close(slot)
            self._out.pop(slot, None)

    def push(self, pieces: dict) -> dict:
        """{slot: codes [1+n_codebooks, k]} -> {slot: audio}: fp32 [k * frame_length] for a slot opened without a rate
        or format; the samples converted so far for one opened with them. The frames of every slot run in one pass
        (a captured graph per bucket, whatever the slots' formats); then every converted slot's samples are
        converted in one fsb_audio_out launch."""
        for slot in pieces:
            st = self._out.get(slot)
            if st is not None and st.counts.done:
                raise ValueError(f"slot {slot}: the stream was flushed")
        out = super().push(pieces)
        conv = [s for s in out if s in self._out]
        if conv:
            with torch.inference_mode(), self.dac._lock, torch.cuda.device(self.dac.device):
                try:
                    ys = audio.OutputStream.push_many([(self._out[s], out[s]) for s in conv])
                except BaseException:
                    for s in conv:
                        self.broken[s] = True
                    raise
            out.update(zip(conv, ys))
        return out

    def flush(self, slot: int) -> torch.Tensor:
        """End the stream of a slot opened with a rate or format: the samples the filter's look-ahead held back (its
        window closed with zeros, as the one-shot conversion closes it). The slot then takes no more pushes until it is
        closed and opened again. A slot opened without either has nothing pending: fp32 [0]."""
        self._check_slot(slot)
        if self.broken[slot]:
            raise ValueError(f"slot {slot}: an earlier push failed, its state is lost; close the slot")
        st = self._out.get(slot)
        if st is None:
            return torch.empty(0, dtype=torch.float32, device=self.dac.device)
        if st.counts.done:
            raise ValueError(f"slot {slot}: the stream was already flushed")
        with torch.inference_mode(), self.dac._lock, torch.cuda.device(self.dac.device):
            try:
                return st.flush()
            except BaseException:
                self.broken[slot] = True
                raise

    def _layer_geometry(self) -> list:
        dac, D = self.dac, self.dac.cfg.latent_dim
        out, r = [], 1
        for u in dac.up:
            out.append((-min(u["conv"].shifts), D, r))
            r *= u["f"]
            out.append((u["cnx"]["k"] - 1, D, r))
        out.append((-min(dac.dec_in.shifts), D, r))
        cin = dac.cfg.decoder_dim
        for blk in dac.dec_blocks:
            out.append((-min(blk["up"].shifts), cin, r))
            r *= blk["stride"]
            cin //= 2
            for ru in blk["res"]:
                assert ru["c1"].taps == 1
                out.append((-min(ru["c7"].shifts), cin, r))
        out.append((dac.dec_out_k - 1, cin, r))
        return out

    def _check_piece(self, slot: int, codes) -> None:
        S_ = self.dac.n_stage
        if codes.ndim != 2 or codes.shape[0] != S_:
            raise ValueError(f"slot {slot}: codes must be [{S_}, k], got {tuple(codes.shape)}")
        if not 1 <= codes.shape[1] <= self.k_max:
            raise ValueError(f"slot {slot}: {codes.shape[1]} frames, a push takes 1 .. {self.k_max}")

    @staticmethod
    def _frames(codes) -> int:
        return int(codes.shape[1])

    def _describe(self, items: list, ks: list, nb: int, kb: int) -> tuple:
        """Host-side description of a push: rows, positions, slots and valid rows per rate; the clamped codes."""
        cfg, S_ = self.dac.cfg, self.dac.n_stage
        scratch = self.slots
        row_seq = [scratch] * (nb * kb)
        row_pos = [j for _ in range(nb) for j in range(kb)]
        slot_of = [-1] * nb
        valid = {r: [0] * nb for r in self.rates}
        for i, ((slot, _), k) in enumerate(zip(items, ks)):
            p = self.pos[slot]
            slot_of[i] = slot
            for j in range(k):
                row_seq[i * kb + j], row_pos[i * kb + j] = slot, p + j
            for r in self.rates:
                valid[r][i] = k * r
        meta_h = torch.tensor(row_seq + row_pos + slot_of + [v for r in self.rates for v in valid[r]],
                              dtype=torch.int32)
        idx_h = torch.zeros(nb, S_, kb, dtype=torch.int32)
        for i, (_, codes) in enumerate(items):
            idx_h[i, :, : ks[i]] = codes.to(device="cpu", dtype=torch.int32)
        idx_h[:, 0].clamp_(min=0, max=cfg.semantic_codebook_size - 1)  # rvq.py:354-359 (on our copy)
        idx_h[:, 1:].clamp_(min=0, max=cfg.codebook_size - 1)
        return idx_h, meta_h

    def _alloc_static(self, nb: int, kb: int, host: tuple) -> tuple:
        return (torch.empty(nb * self.dac.n_stage * kb, dtype=torch.int32, device=self.dac.device),
                torch.empty(host[1].numel(), dtype=torch.int32, device=self.dac.device))

    @staticmethod
    def _stage(st: tuple, items: list, ks: list, host: tuple) -> None:
        st[0].copy_(host[0].reshape(-1))
        st[1].copy_(host[1])

    def _outputs(self, wav: torch.Tensor, items: list, ks: list) -> dict:
        FL = self.dac.frame_length
        return {slot: wav[i, : k * FL].clone() for i, ((slot, _), k) in enumerate(zip(items, ks))}

    def _body(self, nb: int, kb: int, st: tuple, rope_len: int) -> torch.Tensor:
        """The device work of one push (eager or under capture): codes -> transformer (ring K/V) -> upsampler + decoder,
        each conv on a window of its slot's history + the new rows -> waveform [nb, kb * frame_length]."""
        dac, cfg = self.dac, self.dac.cfg
        L, chk = dac.lib, _lib.check
        S_, D = dac.n_stage, cfg.latent_dim
        idx, meta = st
        rows = nb * kb
        row_seq, row_pos, slot_t = meta[:rows], meta[rows: 2 * rows], meta[2 * rows: 2 * rows + nb]
        valid = {r: meta[2 * rows + nb * (1 + j): 2 * rows + nb * (2 + j)] for j, r in enumerate(self.rates)}
        z = dac._buf("pl_z", rows * D)
        chk(L.fsb_codebook_sum(idx.data_ptr(), dac.vq_tab_ptrs.data_ptr(), dac.vq_sizes.data_ptr(), S_, nb, kb, D,
                               z.data_ptr(), _stream()))
        x = dac._transformer(dac.post_tfm, z, nb, kb, "post", kv_cache=self.kv, cache_len=self.ring,
                             rows_at=(row_seq, row_pos), ring=True, rope_len=rope_len)
        window = self._windows(nb, slot_t, valid, "pl_win")

        n = kb
        for i, u in enumerate(dac.up):
            win, H = window(x, n)
            out = dac._buf(f"pl_up_{i}", nb * n * u["f"] * D)
            self._gemm_win(u["conv"], win, nb, H, n, D, out0=out)
            n *= u["f"]
            cn = u["cnx"]
            win, H = window(out, n)
            y = dac._buf("pl_cnx_y", nb * n * D)
            h = dac._buf("pl_cnx_h", nb * n * 4 * D)
            chk(L.fsb_dwconv_ln_window(win.data_ptr(), cn["dw"].data_ptr(), cn["dw_b"].data_ptr(), cn["ln_w"].data_ptr(),
                                       cn["ln_b"].data_ptr(), nb, H + n, H, n, D, cn["k"], 1e-6, y.data_ptr(),
                                       _stream()))
            dac._gemm(cn["pw1"], y, nb, n, D, n, out0=h, act=1)
            dac._gemm(cn["pw2"], h, nb, n, 4 * D, n, out0=out, gamma=cn["gamma"], resid=out)
            x = out
        c = cfg.decoder_dim
        numel = nb * n * c
        for s_ in cfg.decoder_rates:
            numel = max(numel, nb * n * s_ * c // 2)
            n, c = n * s_, c // 2
        n = kb * int(math.prod(cfg.downsample_factor))
        bufs = {k: dac._buf(f"pl_dec_{k}", numel) for k in ("a0", "a1", "x", "m")}
        win, H = window(x, n)
        first = dac.dec_blocks[0]
        self._gemm_win(dac.dec_in, win, nb, H, n, cfg.latent_dim, out1=bufs["a0"], snake=first["s_in"])
        a, spare = "a0", "a1"
        cin = cfg.decoder_dim
        for bi, blk in enumerate(dac.dec_blocks):
            cout = cin // 2
            win, H = window(bufs[a], n)
            self._gemm_win(blk["up"], win, nb, H, n, cin, out0=bufs["x"], out1=bufs[spare], snake=blk["up_snake"])
            a, spare = spare, a
            n *= blk["stride"]
            for j, ru in enumerate(blk["res"]):
                if j < 2:
                    nxt = blk["res"][j + 1]["s0"]
                elif bi + 1 < len(dac.dec_blocks):
                    nxt = dac.dec_blocks[bi + 1]["s_in"]
                else:
                    nxt = dac.dec_out_snake
                win, H = window(bufs[a], n)
                self._gemm_win(ru["c7"], win, nb, H, n, cout, out1=bufs["m"], snake=ru["s1"])
                dac._gemm(ru["c1"], bufs["m"], nb, n, cout, n, out0=bufs["x"] if j < 2 else None, out1=bufs[spare],
                          snake=nxt, resid=bufs["x"])
                a, spare = spare, a
            cin = cout
        win, H = window(bufs[a], n)
        wav = torch.empty(nb, H + n, dtype=torch.float32, device=dac.device)
        chk(L.fsb_final_conv_tanh(win.data_ptr(), dac.dec_out_w.data_ptr(), dac.dec_out_b, nb, H + n, cin,
                                  dac.dec_out_k, wav.data_ptr(), _stream()))
        return wav[:, H:]


class EncodeStreamPool(_StreamPool):
    """Streaming `encode` of up to `slots` independent streams, encoded together; a push computes only the new frames of
    the streams in it: push({slot: waveform fp32 [k * frame_length]}, 1 <= k <= k_max) -> {slot: codes int64
    [n_stages, k]}. A stream's codes, concatenated, are bit-identical to `DAC.encode` of its whole waveform alone (a
    last partial frame is zero-padded by the caller, which is exactly encode's right pad). The encoder is causal from
    end to end, so every layer keeps only what its next rows read:

    * first conv: the last K - 1 = 6 samples of the waveform, kept as 2 rows of 4 fp32 samples (16-byte rows for
      fsb_window_fill / roll) and read by fsb_first_conv_window.
    * encoder ResidualUnits: the dilated k7 conv keeps 6 * dilation rows of its Snake-activated input (6, 18, 54); the
      k1 conv and the residual need none.
    * strided `down` convs (k = 2 * stride, read as [T / stride][stride * C] rows, 2 taps): one row of that view; the
      plain conv GEMM over the window computes them. `enc_out` (k3): 2 rows. The quantizer's downsample convs have
      k = stride (one tap) and need no history. ConvNeXt depthwise convs: 6 rows.
    * transformers: the encoder's (window 512 at 4 rows per frame) and `pre_module` (window 128 at 1 row per frame)
      keep their K/V in rings of R = round_up(window + rows per frame * k_max + 63, 64) positions per slot and layer
      (fsb_qkv_rope_ring / fsb_window_attn_ring), at absolute positions that grow without bound.
    * streams at other sample rates: a slot opened with `open(sample_rate=sr)` takes pieces of any length at `sr` (1-D
      float32, or int16 PCM), and `flush(slot)` ends the stream. Each push resamples the new samples eagerly, before
      the frame pass (fish_speech_b200.audio.StreamResampler, every such slot of the push in one launch), into a
      per-slot carry of fewer than frame_length samples at the codec's rate; the whole frames go through the pass
      below (in rounds of at most k_max frames) and the push returns every frame completed so far, possibly none.
      `flush` pads the last partial frame with zeros, as `encode` pads. The codes are bit-identical to `encode` of the
      whole clip resampled by `audio.resample`.
    * ragged pushes, padding rows, the scratch sequence, graph capture and failed pushes as in DecodeStreamPool, except
      that every window's padding rows are zeroed (fsb_window_fill_zero). The shared window buffer holds other layers'
      rows before (the waveform window's fp32 samples read as bf16 can be Inf or NaN), and the tiled window attention
      adds zero-weighted V rows of every run in a query tile into each row of the tile: a non-finite V in the scratch
      sequence would turn valid rows into NaN, and the vector quantiser a NaN latent into an out-of-range code index.
    """

    _fill = "fsb_window_fill_zero"
    _rs: Mapping = MappingProxyType({})  # replaced per pool; no slot has a rate in a pool built without __init__

    def __init__(self, dac: "DAC", slots: int, k_max: int, n_quantizers: Optional[int], max_graphs: int):
        if slots < 1 or k_max < 1:
            raise ValueError(f"stream pool needs slots >= 1 and k_max >= 1 (got {slots}, {k_max})")
        cfg, FL = dac.cfg, dac.frame_length
        self.dac = dac
        self._rs = {}     # slot -> StreamResampler, for the streams opened with a sample rate
        self._carry = {}  # slot -> their fp32 samples at the codec's rate not yet in a frame (< frame_length)
        self.n_stage = dac.n_stage if n_quantizers is None else min(dac.n_stage, 1 + int(n_quantizers))
        # the transformers in execution order, with their rows per frame; slot `slots` is the scratch sequence
        tfms, r = [], FL
        for blk in dac.enc_blocks:
            r //= blk["stride"]
            if blk["tfm"] is not None:
                tfms.append((blk["tfm"], r))
        tfms.append((dac.pre_tfm, r // int(math.prod(cfg.downsample_factor))))
        self._tfms, self.rings, self.kv_t = [], [], []
        for tf, r in tfms:
            t: TfmConfig = tf["cfg"]
            if not t.window_size or t.window_size <= 0:
                raise ValueError("encode stream pool needs window-limited transformers")
            if (int(slots) * int(k_max) * r > DAC.ONE_SHOT_MAX_ROWS):
                raise ValueError(f"encode stream pool: slots x k_max x {r} transformer rows per frame = "
                                 f"{int(slots) * int(k_max) * r} exceeds the {DAC.ONE_SHOT_MAX_ROWS} rows one launch takes")
            R = _pad64(t.window_size + r * int(k_max) + 63)
            n = (int(slots) + 1) * t.n_head * (R + 64) * t.head_dim
            self._tfms.append((t, r))
            self.rings.append(R)
            self.kv_t.append([(torch.zeros(n, dtype=torch.bfloat16, device=dac.device),
                               torch.zeros(n, dtype=torch.bfloat16, device=dac.device)) for _ in tf["layers"]])
        self.kv = [kv for layers in self.kv_t for kv in layers]
        self.layers = self._layer_geometry()
        super().__init__(dac, slots, k_max, max_graphs)

    def _layer_geometry(self) -> list:
        """(H rows, row width in bf16 units, rows per frame) per windowed layer input, in execution order."""
        dac, cfg = self.dac, self.dac.cfg
        FL = dac.frame_length
        out = [(-(-(dac.enc_in_w.shape[1] - 1) // 4), 8, FL // 4)]  # waveform: rows of 4 fp32 samples
        r, c = FL, cfg.encoder_dim
        for blk in dac.enc_blocks:
            for ru in blk["res"]:
                assert ru["c1"].taps == 1
                out.append((-min(ru["c7"].shifts), c, r))
            s = blk["stride"]
            r //= s
            out.append((-min(blk["down"].shifts), s * c, r))
            c = blk["dim"]
        out.append((-min(dac.enc_out.shifts), c, r))
        for dn in dac.down:
            assert dn["conv"].taps == 1  # kernel = stride: no history
            r //= dn["f"]
            out.append((dn["cnx"]["k"] - 1, cfg.latent_dim, r))
        return out

    def _check_piece(self, slot: int, wav) -> None:
        FL = self.dac.frame_length
        if not isinstance(wav, torch.Tensor) or wav.ndim != 1 or wav.dtype != torch.float32:
            raise ValueError(f"slot {slot}: a piece must be a 1-D float32 waveform")
        if wav.numel() % FL:
            raise ValueError(f"slot {slot}: {wav.numel()} samples is not a whole number of {FL}-sample frames "
                             "(zero-pad the last piece)")
        if not 1 <= wav.numel() // FL <= self.k_max:
            raise ValueError(f"slot {slot}: {wav.numel() // FL} frames, a push takes 1 .. {self.k_max}")

    def _frames(self, wav) -> int:
        return wav.numel() // self.dac.frame_length

    def open(self, sample_rate: Optional[int] = None) -> int:
        """A new stream's slot. Without `sample_rate`, its pushes take whole frames of fp32 audio at the codec's rate;
        with it, pieces of any length at `sample_rate` (1-D float32, or int16 PCM), ended by `flush`."""
        if sample_rate is not None and int(sample_rate) <= 0:
            raise ValueError(f"sample_rate must be positive (got {sample_rate})")
        with self.dac._lock, torch.cuda.device(self.dac.device):
            slot = super().open()
            if sample_rate is not None:
                self._rs[slot] = audio.StreamResampler(int(sample_rate), self.dac.sample_rate, self.dac.device)
                self._carry[slot] = torch.empty(0, dtype=torch.float32, device=self.dac.device)
            return slot

    def close(self, slot: int) -> None:
        with self.dac._lock:
            super().close(slot)
            if slot in self._rs:
                del self._rs[slot], self._carry[slot]

    def push(self, pieces: dict) -> dict:
        """{slot: piece} -> {slot: codes int64 [n_stages, k]}. A slot opened without a sample rate takes 1 .. k_max
        whole frames and gets their k codes; a slot opened with one takes any piece and gets the codes of the frames
        it completed (k >= 0)."""
        if not any(s in self._rs for s in pieces):
            return super().push(pieces)
        for slot, piece in pieces.items():
            self._check_slot(slot)
            if self.broken[slot]:
                raise ValueError(f"slot {slot}: an earlier push failed, its state is lost; close the slot")
            if slot not in self._rs:
                self._check_piece(slot, piece)
            else:
                self._check_rated_piece(slot, piece)
        with self.dac._lock, torch.cuda.device(self.dac.device):
            try:
                frames = self._resample_to_frames({s: p for s, p in pieces.items() if s in self._rs})
                frames.update({s: p for s, p in pieces.items() if s not in self._rs})
                return self._push_frames(frames)
            except BaseException:
                for slot in pieces:
                    self.broken[slot] = True
                raise

    def flush(self, slot: int) -> torch.Tensor:
        """End the stream of a slot opened with a sample rate: the rest of its samples, the last partial frame
        zero-padded as `encode` pads it -> codes int64 [n_stages, k] (k >= 0). The slot then takes no more pushes
        until it is closed and opened again. A slot opened without a rate has nothing pending: [n_stages, 0]."""
        self._check_slot(slot)
        if self.broken[slot]:
            raise ValueError(f"slot {slot}: an earlier push failed, its state is lost; close the slot")
        if slot not in self._rs:
            return torch.empty(self.n_stage, 0, dtype=torch.int64, device=self.dac.device)
        if self._rs[slot].counts.done:
            raise ValueError(f"slot {slot}: the stream was already flushed")
        with self.dac._lock, torch.cuda.device(self.dac.device):
            try:
                return self._push_frames(self._resample_to_frames({slot: None}))[slot]
            except BaseException:
                self.broken[slot] = True
                raise

    def _check_rated_piece(self, slot: int, piece) -> None:
        if not isinstance(piece, torch.Tensor) or piece.ndim != 1 or piece.dtype not in (torch.float32, torch.int16):
            raise ValueError(f"slot {slot}: a piece must be a 1-D float32 waveform or int16 PCM")
        if self._rs[slot].counts.done:
            raise ValueError(f"slot {slot}: the stream was flushed")

    def _resample_to_frames(self, pieces: dict) -> dict:
        """{slot: piece at the slot's rate, or None to flush} -> {slot: the whole frames now complete at the codec's
        rate, fp32 [k * frame_length]}; the rest stays in the slot's carry."""
        FL, dev = self.dac.frame_length, self.dac.device
        todo = []
        for slot, piece in pieces.items():
            x = None
            if piece is not None:
                x = piece.to(dev)
                if x.dtype == torch.int16:
                    x = audio.pcm_to_mono(x, audio.PCM_S16)
            todo.append((self._rs[slot], x))
        frames = {}
        for (slot, piece), y in zip(pieces.items(), audio.StreamResampler.push_many(todo)):
            c = torch.cat((self._carry[slot], y))
            if piece is None:
                c = torch.nn.functional.pad(c, (0, -c.numel() % FL))  # encode's right pad
            k = c.numel() // FL
            frames[slot], self._carry[slot] = c[: k * FL], c[k * FL:]
        return frames

    def _push_frames(self, frames: dict) -> dict:
        """{slot: fp32 [k * frame_length], any k >= 0} -> {slot: codes [n_stages, k]}: pushes of at most k_max frames."""
        FL = self.dac.frame_length
        out = {s: [] for s in frames}
        done = dict.fromkeys(frames, 0)
        while True:
            rnd = {}
            for s, f in frames.items():
                k = min(self.k_max, f.numel() // FL - done[s])
                if k > 0:
                    rnd[s] = f[done[s] * FL: (done[s] + k) * FL]
                    done[s] += k
            if not rnd:
                break
            for s, c in super().push(rnd).items():
                out[s].append(c)
        return {s: torch.cat(v, dim=1) if v else torch.empty(self.n_stage, 0, dtype=torch.int64, device=self.dac.device)
                for s, v in out.items()}

    def _describe(self, items: list, ks: list, nb: int, kb: int) -> torch.Tensor:
        """(sequence, position) of every transformer row, then the slot of each stream and its valid rows per rate."""
        scratch = self.slots
        meta = []
        for _, r in self._tfms:
            n = kb * r
            row_seq = [scratch] * (nb * n)
            row_pos = [j for _ in range(nb) for j in range(n)]
            for i, ((slot, _), k) in enumerate(zip(items, ks)):
                p = self.pos[slot] * r
                for j in range(k * r):
                    row_seq[i * n + j], row_pos[i * n + j] = slot, p + j
            meta += row_seq + row_pos
        slot_of = [slot for slot, _ in items] + [-1] * (nb - len(items))
        meta += slot_of
        for r in self.rates:
            meta += [k * r for k in ks] + [0] * (nb - len(items))
        return torch.tensor(meta, dtype=torch.int32)

    def _alloc_static(self, nb: int, kb: int, meta_h: torch.Tensor) -> tuple:
        # zeros: the padding samples of a ragged push are never read into a valid row, but stay finite
        return (torch.zeros(nb, kb * self.dac.frame_length, dtype=torch.float32, device=self.dac.device),
                torch.empty(meta_h.numel(), dtype=torch.int32, device=self.dac.device))

    @staticmethod
    def _stage(st: tuple, items: list, ks: list, meta_h: torch.Tensor) -> None:
        for i, (_, wav) in enumerate(items):
            st[0][i, : wav.numel()].copy_(wav)
        st[1].copy_(meta_h)

    @staticmethod
    def _outputs(codes: torch.Tensor, items: list, ks: list) -> dict:
        return {slot: codes[i, :, :k].long() for i, ((slot, _), k) in enumerate(zip(items, ks))}

    def _body(self, nb: int, kb: int, st: tuple, rope_len: int) -> torch.Tensor:
        """The device work of one push (eager or under capture): waveform -> encoder -> quantizer downsample ->
        pre_module -> residual VQ, each causal conv on a window of its slot's history + the new rows -> codes int32
        [nb, n_stages, kb]. The layer walk is DAC._encode_one_shot's."""
        dac, cfg = self.dac, self.dac.cfg
        L, chk = dac.lib, _lib.check
        FL, D = dac.frame_length, cfg.latent_dim
        wav, meta = st
        off, rows_at = 0, []
        for _, r in self._tfms:
            rows = nb * kb * r
            rows_at.append((meta[off: off + rows], meta[off + rows: off + 2 * rows]))
            off += 2 * rows
        slot_t = meta[off: off + nb]
        valid = {r: meta[off + nb * (1 + j): off + nb * (2 + j)] for j, r in enumerate(self.rates)}
        window = self._windows(nb, slot_t, valid, "ep_win")
        tfm_at = iter(range(len(self._tfms)))

        def transformer(tf: dict, x: torch.Tensor, T: int) -> torch.Tensor:
            ti = next(tfm_at)
            return dac._transformer(tf, x, nb, T, "", kv_cache=self.kv_t[ti], cache_len=self.rings[ti],
                                    rows_at=rows_at[ti], ring=True, rope_len=rope_len)

        d0 = cfg.encoder_dim
        Tc = kb * FL
        win, H = window(wav, Tc // 4)
        bufs = [dac._buf(f"ep_enc_{k}", nb * Tc * d0) for k in range(3)]
        x, a, m = 0, 1, 2
        r0 = dac.enc_blocks[0]["res"][0]
        chk(L.fsb_first_conv_window(win.data_ptr(), dac.enc_in_w.data_ptr(), dac.enc_in_b.data_ptr(),
                                    r0["s0"].alpha.data_ptr(), r0["s0"].inv.data_ptr(), nb, 4 * H + Tc, 4 * H, Tc, d0,
                                    dac.enc_in_w.shape[1], bufs[x].data_ptr(), bufs[a].data_ptr(), _stream()))
        c = d0
        for bi, blk in enumerate(dac.enc_blocks):
            for j, ru in enumerate(blk["res"]):
                win, H = window(bufs[a], Tc)
                self._gemm_win(ru["c7"], win, nb, H, Tc, c, out1=bufs[m], snake=ru["s1"])
                nxt = blk["res"][j + 1]["s0"] if j < 2 else blk["s_out"]
                dac._gemm(ru["c1"], bufs[m], nb, Tc, c, Tc, out0=bufs[x] if j < 2 else None, out1=bufs[a],
                          snake=nxt, resid=bufs[x])
            s, cout = blk["stride"], blk["dim"]
            Tn = Tc // s
            last = bi + 1 == len(dac.enc_blocks)
            sn = dac.enc_out_snake if last else dac.enc_blocks[bi + 1]["res"][0]["s0"]
            win, H = window(bufs[a], Tn)  # the [Tc / s][s * c] view
            if blk["tfm"] is not None:
                self._gemm_win(blk["down"], win, nb, H, Tn, s * c, out0=bufs[x])
                n_out = transformer(blk["tfm"], bufs[x], Tn)
                chk(L.fsb_snake(n_out.data_ptr(), sn.alpha.data_ptr(), sn.inv.data_ptr(), nb * Tn * cout, cout,
                                bufs[a].data_ptr(), _stream()))
                bufs[x][: nb * Tn * cout].copy_(n_out[: nb * Tn * cout])
            else:
                self._gemm_win(blk["down"], win, nb, H, Tn, s * c, out0=bufs[x], out1=bufs[m], snake=sn)
                a, m = m, a
            Tc, c = Tn, cout
        win, H = window(bufs[a], Tc)
        cur = dac._buf("ep_z", nb * Tc * D)
        self._gemm_win(dac.enc_out, win, nb, H, Tc, c, out0=cur)
        for i, dn in enumerate(dac.down):
            f = dn["f"]
            Tn = Tc // f
            out = dac._buf(f"ep_down_{i}", nb * Tn * D)
            dac._gemm(dn["conv"], cur, nb, Tn, f * D, Tn, out0=out)
            cn = dn["cnx"]
            win, H = window(out, Tn)
            y = dac._buf("ep_cnx_y", nb * Tn * D)
            h = dac._buf("ep_cnx_h", nb * Tn * 4 * D)
            chk(L.fsb_dwconv_ln_window(win.data_ptr(), cn["dw"].data_ptr(), cn["dw_b"].data_ptr(), cn["ln_w"].data_ptr(),
                                       cn["ln_b"].data_ptr(), nb, H + Tn, H, Tn, D, cn["k"], 1e-6, y.data_ptr(),
                                       _stream()))
            dac._gemm(cn["pw1"], y, nb, Tn, D, Tn, out0=h, act=1)
            dac._gemm(cn["pw2"], h, nb, Tn, 4 * D, Tn, out0=out, gamma=cn["gamma"], resid=out)
            cur, Tc = out, Tn
        zq = transformer(dac.pre_tfm, cur, Tc)
        # padding frames belong to no stream: quantise each stream's valid frames only
        codes = torch.empty(nb, self.n_stage, Tc, dtype=torch.int32, device=dac.device)
        chk(L.fsb_vq_encode_valid(zq.data_ptr(), dac.vq_in_w.data_ptr(), dac.vq_in_b.data_ptr(), dac.vq_cbn.data_ptr(),
                                  dac.vq_cb_off.data_ptr(), dac.vq_sizes.data_ptr(), dac.vq_tab_ptrs.data_ptr(),
                                  self.n_stage, cfg.codebook_dim, nb, Tc, D, valid[self._tfms[-1][1]].data_ptr(),
                                  codes.data_ptr(), _stream()))
        return codes


class _SnakeView:
    """Snake parameters repeated for the (p, co) channel order of a transposed-conv GEMM."""

    def __init__(self, s: _Snake, repeat: int):
        self.alpha = s.alpha.repeat(repeat).contiguous()
        self.inv = s.inv.repeat(repeat).contiguous()
