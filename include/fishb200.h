/* fishb200 — C-ABI of the H100-native (sm_90a) Fish-Speech inference hot path.
 *
 * The reference (fishaudio/fish-speech @ 3dd1f85c) is pure Python/PyTorch and has no FFI of its own:
 * its boundary for this path is the Python API listed in SURVEY.md §8(b).  This header is what a
 * maintainer's `ctypes` stub binds instead of the eager PyTorch modules; every entry point names the
 * reference symbol (file:line under the reference checkout) whose work it replaces.  See
 * INTEGRATION.md for the reference-side binding.
 *
 * Conventions: plain pointers and sizes only (no torch types).  All `d_` pointers are CUDA device
 * pointers owned by the caller and must stay valid for the lifetime of the handle they are given to;
 * `h_` pointers are host memory.  Every function returns 0 on success, non-zero on failure with the
 * message available from fsb_last_error() (per host thread).  `stream` is a cudaStream_t passed as
 * void*.  Handles are not thread-safe; distinct handles may be driven from different host threads
 * (the reference runs the LM worker thread and the codec caller concurrently:
 * fish_speech/models/text2semantic/inference.py:748-799).
 */
#ifndef FISHB200_H
#define FISHB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* fsb_last_error(void);
/* Number of kernels this host thread has launched through the library (bench.py: gpu_launches). */
long long fsb_launch_count(void);
int fsb_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* cudaMemcpy helpers so Python hosts need no CUDA bindings of their own. */
int fsb_memcpy_d2h(void* h_dst, const void* d_src, size_t bytes, void* stream);
int fsb_memcpy_h2d(void* d_dst, const void* h_src, size_t bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dual-AR text2semantic transformer
 *   replaces DualARTransformer.forward_generate / forward_generate_fast
 *     (fish_speech/models/text2semantic/llama.py:390-466, 799-828) and
 *   decode_one_token_ar / decode_n_tokens / the prefill call in generate
 *     (fish_speech/models/text2semantic/inference.py:96-181, 184-238, 322-335).
 * ---------------------------------------------------------------------------------------------- */
typedef struct fsb_lm fsb_lm;

typedef struct {
    /* slow (time-axis) stack: BaseModelArgs, llama.py:28-73 */
    int dim, n_layer, n_head, n_kv_head, head_dim, intermediate;
    /* fast (codebook-axis) stack: DualARModelArgs, llama.py:156-193 */
    int fast_dim, n_fast_layer, fast_n_head, fast_n_kv_head, fast_head_dim, fast_intermediate;
    int vocab_size, codebook_size, num_codebooks;
    int semantic_begin_id, semantic_end_id, im_end_id;
    float norm_eps;
    int qk_norm, fast_qk_norm;           /* attention_qk_norm / fast_attention_qk_norm */
    int scale_codebook_embeddings;       /* llama.py:416-420 */
    int norm_fastlayer_input;            /* llama.py:459-461 */
    int max_batch;                       /* resident sequences ("slots"), <= 64; above 32 the decode step runs
                                            its 64-row tile (RT = 64), else the 32-row one (RT = 32) */
    int kv_len;                          /* KV-cache positions per sequence (its capacity) */
    int max_rows;                        /* token rows per prefill pass */
    int max_frames;                      /* generated frames kept per sequence */
    int debug;                           /* keep logits / per-layer activations for tests */
    int kv_pages;                        /* slow KV cache pool, in pages of 64 positions (every slow layer, K and V:
                                            64 x 2 x n_layer x n_kv_head x head_dim x 2 B); 0 = max_batch x
                                            ceil(kv_len / 64), room for every slot at full capacity. Sequences map
                                            pages through the "kv_page" table (fsb_lm_buffer), which the caller
                                            fills: a position whose page is not mapped is neither written nor read */
    int attn_split;                      /* 0 = off. Otherwise positions per span of the decode attention, a multiple
                                            of 64: a slow-stack row whose context is longer than this has its history
                                            split into spans of this many positions (edges at absolute positions), one
                                            CTA each, merged in ascending order by a kernel of its own, so that one
                                            long request does not set the frame time of every slot. Such a row's bits
                                            depend on its own history only (not on slot, neighbours or context bound)
                                            but differ in the last places from the unsplit kernel's; rows up to this
                                            length, and every frame whose context bound is at most this, keep today's
                                            kernel and bits. At most what one span's scores fit in shared memory
                                            (10 944 at head_dim 128 with 4 query heads per KV head) */
} fsb_lm_config;

/* One TransformerBlock (llama.py:831-987). bf16, row-major [out_features, in_features]. */
typedef struct {
    const void* d_attn_norm;  /* [dim] */
    const void* d_wqkv;       /* [(H+2Hkv)*Dh, dim] */
    const void* d_bqkv;       /* optional */
    const void* d_q_norm;     /* [Dh] optional */
    const void* d_k_norm;     /* [Dh] optional */
    const void* d_wo;         /* [dim, H*Dh] */
    const void* d_bo;         /* optional */
    const void* d_ffn_norm;   /* [dim] */
    const void* d_w13;        /* [ceil(I/64)*128, dim]: w1 and w3 interleaved per 128-row tile so that SwiGLU runs in
                                 the GEMM epilogue: tile t holds hidden features [64t, 64t+64); inside it, row
                                 32w + l (l < 16) = w1[64t + 16w + l] and row 32w + 16 + l = w3[64t + 16w + l];
                                 rows past I are zero (fish_speech_b200.engine.interleave_w13 builds it) */
    const void* d_w2;         /* [dim, I] */
} fsb_lm_layer;

typedef struct {
    const void* d_embeddings;           /* [vocab, dim] */
    const void* d_codebook_embeddings;  /* [num_codebooks*codebook_size, dim] */
    const void* d_norm;                 /* [dim] */
    const void* d_head;                 /* [head_rows, dim]: the rows of the (tied) LM head that the
                                           semantic_logit_bias leaves selectable — semantic ids in
                                           order, then <|im_end|> (inference.py:308-320) */
    int head_rows;                      /* (semantic_end_id - semantic_begin_id + 1) + 1 */
    const void* d_freqs;                /* bf16 [kv_len, head_dim/2, 2] (llama.py:1004-1023) */
    const fsb_lm_layer* layers;         /* host array [n_layer] */
    const void* d_fast_embeddings;      /* [codebook_size, fast_dim] */
    const void* d_fast_norm;            /* [fast_dim] */
    const void* d_fast_output;          /* [codebook_size, fast_dim] */
    const void* d_fast_freqs;           /* bf16 [num_codebooks, fast_head_dim/2, 2] */
    const void* d_fast_proj_w;          /* optional [fast_dim, dim] (llama.py:665-668) */
    const void* d_fast_proj_b;          /* optional [fast_dim] */
    const fsb_lm_layer* fast_layers;    /* host array [n_fast_layer] */
} fsb_lm_weights;

/* sample() parameters (inference.py:54-93).  temperature / top_p must already be rounded to the
 * model dtype the way the reference builds them (torch.tensor(v, dtype=bf16), inference.py:303-304).
 * top_k <= 1 keeps the most likely candidate only (greedy, no RAS re-draw), as the reference's mask does for any
 * top_k <= 1; a top_k above 256 samples exactly as 256 (see INTEGRATION.md). */
typedef struct {
    float temperature;
    float top_p;
    int top_k;
    unsigned long long seed;
} fsb_sampling;

int fsb_lm_create(const fsb_lm_config* cfg, const fsb_lm_weights* w, fsb_lm** out);
void fsb_lm_destroy(fsb_lm* h);

/* Prefill = decode_one_token_ar on whole prompts (inference.py:322-335), for `nseq` sequences packed
 * as `rows` token rows: d_tokens[row][0] = token id, [1..C] = codes; d_row_slot / d_row_pos give the
 * sequence slot and position of each row.  If do_sample != 0 the first frame of each sequence is
 * sampled from its last row (d_last_rows[k], slot d_slots[k]) and stored as output frame 0. */
int fsb_lm_prefill(fsb_lm* h, const int32_t* d_tokens, const int32_t* d_row_slot,
                   const int32_t* d_row_pos, int rows, const int32_t* d_last_rows,
                   const int32_t* d_slots, int nseq, int do_sample, const fsb_sampling* s,
                   void* stream);

/* Fused admission: fsb_lm_prefill with do_sample set, except that the sequences' first frames are not run here. Each
 * sequence's last prompt row (its residual row and sums of squares) and position are staged for its slot d_slots[k]
 * (h_slots[k] on the host: the same list), the slot is marked pending and parked at position -1. The next
 * fsb_lm_decode runs its first frame with a splice after the slow stack that puts each pending slot's staged row into
 * its decode row, and samples a row whose slot has produced no frame yet by the prefill's rule (no RAS); every request
 * gets the tokens fsb_lm_prefill with do_sample would have given it, one fewer pass over the head and fast weights per
 * admission. Needs slot control. A split prompt (longer than max_rows) defers with the call of its last rows; earlier
 * pieces go through fsb_lm_prefill with do_sample = 0. While a slot is pending, fsb_lm_slot_save refuses it and
 * fsb_lm_slot_restore into it drops the pending first frame; fsb_lm_decode needs every pending slot in [0, batch). */
int fsb_lm_prefill_deferred(fsb_lm* h, const int32_t* d_tokens, const int32_t* d_row_slot, const int32_t* d_row_pos,
                            int rows, const int32_t* d_last_rows, const int32_t* d_slots, int nseq,
                            const int32_t* h_slots, void* stream);

/* decode_n_tokens (inference.py:184-238): `nframes` more frames for slots [0, batch). One frame =
 * slow step + constrained sampling (+RAS) + num_codebooks fast steps; captured as a CUDA graph when
 * use_graph != 0. The per-frame <|im_end|> test is kept on the device (finished flags). After
 * fsb_lm_prefill_deferred, the first frame is the fused one (its own graph). */
int fsb_lm_decode(fsb_lm* h, int batch, int nframes, const fsb_sampling* s, int use_graph,
                  void* stream);

/* Row tile of the decode frames. An engine of 33..64 slots holds the step GEMM plans of both tiles: the 64-row plans
 * and 32-row plans with the same stream-K schedule over the first 32 rows of the same buffers (fsb_lm_create fails if
 * the schedules differ). fsb_lm_decode runs a frame of batch <= 32 rows on the 32-row plans and a larger one on the
 * 64-row plans; every output element is the same sum of the same MMAs at either tile, so only the time differs.
 * Decode graphs are kept per (batch, tile, context bound, slot control, fused first frame, noise, sampling), up to 16
 * per engine, so changing the row count or the tile between calls replays a captured frame once it has been seen.
 * fsb_lm_set_decode_tile (test hook): 0 = by the row count (default), 32 or 64 = that tile for every frame (64 needs
 * an engine of more than 32 slots; a decode of more rows than a forced 32-row tile holds fails).
 * fsb_lm_decode_tile: the tile of the last fsb_lm_decode call (0 before the first). fsb_lm_graph_captures: decode
 * frames captured into graphs since fsb_lm_create. */
int fsb_lm_set_decode_tile(fsb_lm* h, int tile);
int fsb_lm_decode_tile(fsb_lm* h);
long long fsb_lm_graph_captures(fsb_lm* h);

/* Prefix KV reuse (SURVEY §8(f).2; the reference re-prefills the whole growing conversation for every chunk,
 * inference.py:611-721). The slow KV cache of a slot stays valid for the positions a prefill wrote until they are
 * overwritten, so a prompt that shares its first p rows with what a slot already holds only needs rows [p, T):
 * call fsb_lm_prefill with d_row_pos starting at p. fsb_lm_copy_kv makes the K/V of positions [0, n_pos) of
 * `src_slot` available in `dst_slot` (every layer, every KV head) for requests that share a system / reference
 * prompt with another slot. Prefill is row-independent, so reused K/V is bit-identical to recomputed K/V. */
int fsb_lm_copy_kv(fsb_lm* h, int src_slot, int dst_slot, int n_pos, void* stream);

/* With the paged slow cache (fsb_lm_config.kv_pages), fsb_lm_copy_kv copies page by page through the "kv_page" table:
 * dst_slot must already map pages of its own (mapped by no other slot) for positions [0, n_pos). A block whose source
 * or destination page is not mapped is skipped; a page both slots map is left as it is. */

/* Copy-on-write of a partly shared page: positions [0, n_pos) (n_pos <= 64) of page `src_page` into page `dst_page`,
 * every slow layer, K and V. fsb_lm_copy_kv above copies through the page table the same way, page by page; both
 * are stream-ordered with the prefill / decode calls. */
int fsb_lm_copy_kv_page(fsb_lm* h, int src_page, int dst_page, int n_pos, void* stream);

/* Upper bound of (position + 1) over all slots for the calls that follow (prompt length + frames decoded so
 * far). Sizes the attention score buffer and, with attn_split, the number of spans launched (a row longer than the
 * bound would lose its last spans); must be set before prefill / decode whenever it grows. */
int fsb_lm_set_context_bound(fsb_lm* h, int max_positions);

/* Per-slot request control — continuous batching over the KV slots, i.e. the batched form of the loop
 * in decode_n_tokens / generate (inference.py:184-359) that the reference runs for one request at a
 * time behind launch_thread_safe_queue (inference.py:748-799). When enabled, prefill and decode ignore
 * `s` (may be NULL) and read, per slot, the device arrays
 *   "slot_state" int32 (0 idle, 1 active, 2 finished, 3 finishing), "slot_limit" int32 (frames allowed,
 *   the prefill's frame included), "slot_temperature" f32, "slot_top_p" f32 (both already rounded to
 *   bf16 by the host, as the reference's tensors are), "slot_top_k" int32 (any value: <= 1 is greedy, as in
 *   fsb_sampling), "slot_seed" uint64.
 * The host writes them (fsb_lm_buffer) before prefilling a request into a slot; the frame kernels stop
 * a slot on <|im_end|> (from its second frame on) or at its limit, freeze its position and counters,
 * and set state = 2; the host collects "out_tokens"[slot][:, :n_out[slot]] and sets the state to 0.
 * The random stream of a request depends on (seed, own frame index, draw) only: a request produces
 * the same tokens alone or with any neighbours, in any slot. */
int fsb_lm_set_slot_control(fsb_lm* h, int enable);

/* Take a running request out of its slot between two decode frames and put it back later, into any slot, with the
 * same bits (slot control must be enabled). fsb_lm_slot_save gathers what the frames keep per slot between frames
 * (the slot-control arrays, frame counter, position, finished flag, RAS window, the last frame's tokens and
 * "out_tokens"[slot][:, :n_out]) into a device blob of fsb_lm_slot_blob_bytes bytes (16-byte aligned), and parks the
 * slot: state 0, position -1, so the frames that follow neither attend for the row nor write its K/V.
 * fsb_lm_slot_restore scatters a blob into `slot`. Each is one small kernel on `stream`; the decode graph stays valid.
 * The slow K/V is not part of the blob: it stays in the pages the slot mapped ("kv_page"), and the caller maps those
 * pages into the slot it restores to. A blob is valid for the handle that wrote it. */
size_t fsb_lm_slot_blob_bytes(fsb_lm* h);
int fsb_lm_slot_save(fsb_lm* h, int slot, void* d_blob, void* stream);
int fsb_lm_slot_restore(fsb_lm* h, int slot, const void* d_blob, void* stream);

/* Reset per-slot generation state (frame counters, RAS window, finished flags, slot states). */
int fsb_lm_reset(fsb_lm* h, void* stream);

/* Named device buffers of the handle, for reading results and for tests:
 *   "out_tokens" int32 [max_batch][C+1][max_frames], "n_out" int32 [max_batch], "pos" int32 [RT],
 *   "step" uint64 [1] (frames decoded since fsb_lm_reset: the Philox counter of the per-call sampling parameters),
 *   "finished" int32 [max_batch], "cur_tok" int32 [max_batch][C+1], "ras_window" int32 [max_batch][10],
 *   the slot-control arrays listed at fsb_lm_set_slot_control, "kv_page" int32 [max_batch][ceil(kv_len / 64)]
 *   (page of each 64-position block of each slot, -1 = not mapped; read by the kernels at run time, so a captured
 *   decode graph stays valid when the caller remaps pages between calls),
 *   "kv_miss" int32 [max_batch] (0, or 1 + the position of a slot's live decode row the first time the slow-stack
 *   decode attention found a page it reads or appends to unmapped: that row attended to nothing and its tokens are
 *   void; zeroed at create, never cleared by the library: the caller zeroes a slot's entry when it reuses the slot),
 *   debug only: "slow_logits" f32 [max_batch][head_rows], "fast_logits" f32 [C][max_batch][codebook_size];
 *   the decode state (for fsb_lm_test_layer_gemms), RT = the decode row tile (32 for max_batch <= 32, else 64):
 *   "x_slow" / "x_fast" bf16 [RT][dim] / [RT][fast_dim] residual streams, "ssq_slow" / "ssq_fast" f32 [RT][32] their
 *   per-128-feature sums of squares, "q" bf16 [RT * max H*Dh] (attn_split only: the finished q heads of the rows
 *   that are split, rows at stride H*Dh) and "attn_span_ws" f32 [max_batch][n_kv_head][spans of the launch]
 *   [G*(head_dim+2)] (attn_split only: per span acc[G][head_dim], max[G], sum[G]; G = n_head / n_kv_head), "attn" bf16 [RT * max H*Dh] (the wo operand: rows of the stack being run at
 *   stride H*Dh), "ffn_h" bf16 [RT * max I] (the w2 operand: rows at stride I of the stack being run);
 *   the KV caches (for fsb_lm_test_layer_attn and the copy tests): "k_slow" / "v_slow" bf16
 *   [n_layer][kv_pages][n_kv_head][64][head_dim] (the page pool), "k_fast" / "v_fast" bf16
 *   [n_fast_layer][max_batch][fast_n_kv_head][num_codebooks][fast_head_dim] (one contiguous block per slot);
 *   the prefill workspaces (for fsb_lm_test_prefill_stage), R = max(max_rows, 128) token rows: "x_prefill" /
 *   "xn_prefill" bf16 [R][dim] (the residual stream and its normed copy, the next GEMM's operand), "q_prefill" bf16
 *   [R][n_head][head_dim], "attn_prefill" bf16 [R][n_head*head_dim], "h_prefill" bf16 [R][intermediate] and
 *   "ws_prefill" f32, flat: the fp32 result of the prefill GEMM run last, [rows][n_out] at a row stride of n_out
 *   ((n_head + 2 n_kv_head) * head_dim for qkv, dim for wo and w2, ceil(intermediate / 64) * 128 for w1|w3, whose
 *   columns are in the interleaved row order of the fused matrix);
 *   the frame-tail buffers (for fsb_lm_test_frame_stage): "fast_hidden" bf16 [RT * max(dim, fast_dim)] (the
 *   fast_project_in operand, rows at stride dim), and fused admission's staged rows "first_frame_x" bf16
 *   [max_batch][dim], "first_frame_ssq" f32 [max_batch][32], "first_frame_pos" int32 [max_batch] and
 *   "first_frame_pending" int32 [max_batch] */
int fsb_lm_buffer(fsb_lm* h, const char* name, void** d_ptr, size_t* bytes);

/* Measurement hook for bench.py: launch every weight-streaming step GEMM of one decode frame `reps` times
 * (no attention / sampling kernels; the finalize kernels run and overwrite the decode state, so call it after
 * the timed generation); returns the algorithmic weight bytes and launch count of one repetition. */
int fsb_lm_bench_gemms(fsb_lm* h, int reps, double* weight_bytes_per_rep, int* launches_per_rep,
                       void* stream);

/* Measurement hook for tools/step_gemm_boundaries.py: the slow stack's step GEMMs of ONE kind (0 = qkv, 1 = wo,
 * 2 = w1|w3, 3 = w2), layers 0..n_layer-1, `reps` times back to back through the decode path's own plans, each with
 * the finalize kernel in front of it (finalize != 0) or without. Returns the weight bytes and launches of one
 * repetition. Overwrites the decode state, like fsb_lm_bench_gemms. */
int fsb_lm_bench_step_kind(fsb_lm* h, int kind, int reps, int finalize, double* weight_bytes_per_rep,
                           int* launches_per_rep, void* stream);

/* Test hook for bit-exact parity of the STOCHASTIC sampler with the reference's torch RNG stream
 * (inference.py:43-46 multinomial_sample_one_no_sync, :114-144 RAS): when d_u != NULL, slot 0 takes the uniforms
 * of draw d of frame f from d_u[(f * draws_per_frame + d) * ld + candidate] (f = frames produced since
 * fsb_lm_reset; d = 0 slow token, 1 slow RAS re-draw, 2p fast codebook p; candidate = restricted head row /
 * code) instead of the library's Philox stream, and forms -log(U) and the scores in bf16 like the reference's
 * tensors. Pass NULL to restore the Philox stream. */
int fsb_lm_set_sampler_noise(fsb_lm* h, const float* d_u, int draws_per_frame, int ld);

/* ------------------------------------------------------------------------------------------------
 * Codec ("Firefly VQ-GAN" = modified Descript-DAC) operators
 *   replace DAC.from_indices / DAC.encode and everything under them
 *     (fish_speech/models/dac/modded_dac.py:874-946, fish_speech/models/dac/rvq.py:293-366).
 * Activations are channels-last bf16 [B][T][C]. The host mirror (fish_speech_b200/models/dac/) walks the
 * reference's module tree and issues one call per layer; weight-norm is folded once at load.
 * ---------------------------------------------------------------------------------------------- */
/* Conv1d / ConvTranspose1d / Linear as a tcgen05 multi-tap implicit-im2col GEMM with fused epilogue:
 *   out[b][t][co] = epi( sum_tap sum_ci x[b][t + shifts[tap]][ci] * w[co][tap*kpad + ci] )
 * rows outside [0, T_in) read as zero (= CausalConvNet's left pad, modded_dac.py:546-552).
 * epi: +bias[co]; GELU if act==1; *gamma[co]; +resid[b][t][co]; tanh if act==2; out0 = value,
 * out1 = Snake(value; alpha[co]) (dac.nn.layers.Snake1d) for the consuming layer. */
int fsb_conv_gemm(const void* d_x, int B, int T_in, int C_in, int row_stride, long long batch_stride,
                  const void* d_w, int C_out, int taps, int kpad, const int* shifts, int T_out,
                  const float* d_bias, const float* d_gamma, const void* d_resid, int act,
                  void* d_out0, void* d_out1, const float* d_alpha, const float* d_inv_alpha, int out_f32,
                  void* stream);
/* ws[row][n] (fp32) = sum_k x[row][k] * w[n][k] — feeds the transformer glue below. */
int fsb_linear_f32(const void* d_x, int rows, int K, const void* d_w, int N, float* d_ws, void* stream);
/* z[b][t][:] = tab_0[idx[b][0][t]] + sum_{c>=1} tab_c[idx[b][c][t]]  (rvq.py:352-363; tab_c =
 * out_proj_c(codebook_c), fp32 [size_c][D]); indices are clamped to the table size like the reference. */
int fsb_codebook_sum(const int32_t* d_idx, const float* const* d_tabs, const int32_t* d_sizes, int ncb, int B,
                     int T, int D, void* d_out, void* stream);
/* ConvNeXt front: causal depthwise conv (k taps) + LayerNorm (rvq.py:176-179). w fp32 [C][K]. */
int fsb_dwconv_ln(const void* d_x, const float* d_w, const float* d_bias, const float* d_ln_w, const float* d_ln_b,
                  int B, int T, int C, int K, float eps, void* d_y, void* stream);
/* Decoder tail: conv K taps C->1 on the Snake'd activation + tanh -> fp32 waveform (modded_dac.py:793-797). */
int fsb_final_conv_tanh(const void* d_a, const float* d_w, float bias, int B, int T, int C, int K, float* d_wav,
                        void* stream);
/* Encoder head: conv K taps 1->C on the fp32 waveform (modded_dac.py:683); raw and/or Snake'd output. */
int fsb_first_conv(const float* d_wav, const float* d_w, const float* d_bias, const float* d_alpha,
                   const float* d_inv_alpha, int B, int T, int C, int K, void* d_raw, void* d_act, void* stream);
/* fsb_first_conv over a stream window (EncodeStreamPool): output sample t of batch item b reads samples
 * origin + t - (K-1) .. origin + t of d_wav [B][T_in] (fp32), so the origin samples before it are its carried history;
 * outputs [B][T_out][C]. origin + T_out <= T_in; at least one of d_raw / d_act. */
int fsb_first_conv_window(const float* d_wav, const float* d_w, const float* d_bias, const float* d_alpha,
                          const float* d_inv_alpha, int B, int T_in, int origin, int T_out, int C, int K, void* d_raw,
                          void* d_act, void* stream);
int fsb_snake(const void* d_x, const float* d_alpha, const float* d_inv_alpha, long long n, int C, void* d_y,
              void* stream);
/* One decoder ResidualUnit -- y = x + conv1(snake_1(conv7_dilated(a))), a = snake_0(x) -- as ONE kernel (dac
 * ResidualUnit, modded_dac.py:599-620 causal variant): the intermediate stays in shared memory. d_a / d_x bf16
 * [B][T][C]; d_w7 [C][7][pad64(C)], d_w1 [C][pad64(C)] bf16 (the packing of fsb_conv_gemm); out0 = y (may alias d_x,
 * may be NULL), out1 = snake_next(y) (must not alias d_a). C in {96, 192, 384} (fsb_res_unit_supported). */
int fsb_res_unit_supported(int C);
int fsb_res_unit(const void* d_a, const void* d_x, int B, int T, int C, int dilation, const void* d_w7,
                 const float* d_b7, const float* d_alpha1, const float* d_inv1, const void* d_w1, const float* d_b1,
                 void* d_out0, void* d_out1, const float* d_alpha_n, const float* d_inv_n, void* stream);
/* 1 semantic + n residual vector-quantiser stages per latent frame (rvq.py:304-317, dac VectorQuantize). */
int fsb_vq_encode(const void* d_z, const float* d_in_w, const float* d_in_b, const float* d_cbn,
                  const int32_t* d_cb_off, const int32_t* d_sizes, const float* const* d_tabs, int S, int cd, int B,
                  int T, int D, int32_t* d_codes, void* stream);
/* fsb_vq_encode of the first d_valid[b] frames of each batch item only (EncodeStreamPool: the frames after them are
 * padding and may hold values that are not finite); the codes of the other frames are not written. */
int fsb_vq_encode_valid(const void* d_z, const float* d_in_w, const float* d_in_b, const float* d_cbn,
                        const int32_t* d_cb_off, const int32_t* d_sizes, const float* const* d_tabs, int S, int cd,
                        int B, int T, int D, const int32_t* d_valid, int32_t* d_codes, void* stream);
/* WindowLimitedTransformer glue (modded_dac.py:174-346) on fp32 GEMM results. */
int fsb_resid_scale_norm(const float* d_y, int ld, const void* d_scale, const void* d_x_in, void* d_x_out,
                         const void* d_norm_w, void* d_n_out, int rows, int D, float eps, int round_bf16,
                         void* stream);
int fsb_qkv_rope(const float* d_qkv, int rows, int H, int Hkv, int Dh, const void* d_freqs, const int32_t* d_row_seq,
                 const int32_t* d_row_pos, void* d_q, void* d_k, void* d_v, int S, void* stream);
int fsb_window_attn(const void* d_q, const void* d_k, const void* d_v, const int32_t* d_row_seq,
                    const int32_t* d_row_pos, int rows, int H, int Hkv, int Dh, int S, int window, void* d_out,
                    void* stream);
int fsb_swiglu_f32(const float* d_y, int rows, int I, void* d_h, void* stream);
/* The same K/V append and window attention over a RING cache when ring != 0 (streaming decode of unbounded length):
 * per (sequence, KV head) S + 64 rows, S a multiple of 64; position p (any p >= 0) is row p % S and rows [0, 64) are
 * mirrored in rows [S, S + 64). Only the latest S positions are kept, so the attention needs 0 < window < S and
 * S >= window + (positions appended per sequence in one call) - 1. Same terms in the same order as over a linear cache:
 * the results are bit-identical to fsb_qkv_rope / fsb_window_attn with a cache long enough to hold every position.
 * head_dim 64 or 128. ring == 0: exactly fsb_qkv_rope / fsb_window_attn. */
int fsb_qkv_rope_ring(const float* d_qkv, int rows, int H, int Hkv, int Dh, const void* d_freqs,
                      const int32_t* d_row_seq, const int32_t* d_row_pos, void* d_q, void* d_k, void* d_v, int S,
                      int ring, void* stream);
int fsb_window_attn_ring(const void* d_q, const void* d_k, const void* d_v, const int32_t* d_row_seq,
                         const int32_t* d_row_pos, int rows, int H, int Hkv, int Dh, int S, int window, int ring,
                         void* d_out, void* stream);
/* Per-layer stream windows (DecodeStreamPool, EncodeStreamPool): a layer's input is viewed per stream as [H + n][row] with rows 0..H-1
 * its carried causal history. fsb_window_fill writes win [nb][H + n][row]: rows 0..H-1 from state [slots][H][row] at
 * d_slot[i], rows H..H+d_valid[i]-1 from the producer's dense output [nb][n][row]; other rows are left as they are
 * (padding after the valid rows). fsb_window_roll writes the last H valid rows (window rows d_valid[i] ..
 * d_valid[i]+H-1) back to the slot's state. A negative slot skips the stream. row_bytes a multiple of 16. */
int fsb_window_fill(const void* d_state, const void* d_dense, void* d_win, const int32_t* d_slot,
                    const int32_t* d_valid, int nb, int H, int n, int row_bytes, void* stream);
/* fsb_window_fill that also zeroes every row it does not fill: the rows past a stream's valid rows, and all rows of a
 * stream with a negative slot (EncodeStreamPool). Padding rows then never hold what the buffer held before, which may
 * not be finite: the window attention multiplies a row's zero weights by the V rows of every run in its query tile, so
 * a non-finite V in the scratch sequence would reach valid rows. */
int fsb_window_fill_zero(const void* d_state, const void* d_dense, void* d_win, const int32_t* d_slot,
                         const int32_t* d_valid, int nb, int H, int n, int row_bytes, void* stream);
int fsb_window_roll(const void* d_win, void* d_state, const int32_t* d_slot, const int32_t* d_valid, int nb, int H,
                    int n, int row_bytes, void* stream);
/* fsb_dwconv_ln over such a window: output row t = input row origin + t of x [B][T_in][C] (its history = the rows
 * before it); y [B][T_out][C]. origin + T_out <= T_in. */
int fsb_dwconv_ln_window(const void* d_x, const float* d_w, const float* d_bias, const float* d_ln_w,
                         const float* d_ln_b, int B, int T_in, int origin, int T_out, int C, int K, float eps, void* d_y,
                         void* stream);

/* ------------------------------------------------------------------------------------------------
 * Codec input front end (csrc/audio_kernels.cu): PCM at any sample rate -> the codec's mono fp32 input on the device.
 *   replaces the numpy conversion + down-mix and torchaudio.functional.resample of the readers feeding DAC.encode
 *   (tools/vqgan/extract_vq.py:108, fish_speech/models/text2semantic/inference.py:428).
 * Descriptors are arrays in device memory, one per clip; a launch covers many clips (blockIdx.y = clip).
 * ---------------------------------------------------------------------------------------------- */
#define FSB_PCM_S16 0 /* little-endian int16:  x / 32768 */
#define FSB_PCM_S32 1 /* little-endian int32:  x / 2147483648 */
#define FSB_PCM_U8 2  /* unsigned 8-bit:       (x - 128) / 128 */
#define FSB_PCM_F32 3 /* float32 as is */

typedef struct {
    long long src_off;  /* byte offset of the clip's first frame in d_src (any alignment) */
    long long frames;   /* frames of `channels` interleaved samples */
    long long channels;
    long long format;   /* FSB_PCM_* */
    long long dst_off;  /* element offset of the clip's mono output in d_dst */
} fsb_pcm_clip;

/* Mono fp32 of each clip: per frame the channel values (converted in fp32 as above) summed in order from 0.f, then
 * divided by the channel count -- bit-identical to numpy's `x.astype(float32) / scale` and `.mean(axis=1)`.
 * max_frames >= every clip's frames. */
int fsb_pcm_to_mono(const void* d_src, const fsb_pcm_clip* d_clips, int B, long long max_frames, float* d_dst,
                    void* stream);

typedef struct {
    long long x_off;    /* element offset in d_x of input sample x_start of the clip */
    long long x_start;  /* d_x holds the clip's samples [x_start, x_end) from x_off on; samples < 0 or >= x_end are 0 */
    long long x_end;
    long long j0;       /* first output (absolute index in the clip's output) to compute */
    long long out_off;  /* element offset in d_out of output j0 */
    long long n_out;    /* outputs computed: j0 .. j0 + n_out - 1 */
    long long n_fill;   /* elements written from out_off: the n_out outputs, then zeros (>= n_out) */
    const float* w;     /* fp32 [taps][new_rate]: the non-zero taps of each phase; NULL = orig == new (a copy) */
    const int32_t* span;/* int32 [new_rate][2]: phase p's first input offset from q * orig, and its tap count */
    long long orig, new_rate; /* the two rates divided by their gcd */
} fsb_resample_clip;

/* torchaudio.functional.resample(x, orig, new) with its defaults (sinc_interp_hann, lowpass_filter_width 6,
 * rolloff 0.99): output j = q * new + p is sum_m w[m][p] * x(q * orig + span[p][0] + m), m ascending over span[p][1]
 * taps, fp64 fma from 0.0, rounded to fp32 once. The table is built by fish_speech_b200/audio.py. An output's bits depend only on the
 * samples it reads, so a batch, a clip alone and a stream window that holds those samples agree bitwise. */
int fsb_resample(const float* d_x, const fsb_resample_clip* d_clips, int B, long long max_fill, float* d_out,
                 void* stream);

/* ------------------------------------------------------------------------------------------------
 * Codec output front end (csrc/audio_kernels.cu): the decoder's fp32 44.1 kHz waveform -> the client's rate and sample
 * format, on the device, in one pass.
 *   replaces the per-segment `(audio * 32768).astype(np.int16)` of the serving shell (tools/server/inference.py:32-33)
 *   and any resampling a client would do on the host.
 * ---------------------------------------------------------------------------------------------- */
#define FSB_OUT_F32 0   /* float32: the fp32 value y itself */
#define FSB_OUT_PCM16 1 /* int16: trunc(min(max(y, -1), 1) * 32767.0f), the product rounded to nearest (not fused);
                           NaN -> 0. Equal to inference_engine/utils.py:pcm16. */
#define FSB_OUT_MULAW 2 /* uint8: G.711 mu-law (bias 132, 8 segments) of that int16, as audioop.lin2ulaw */

typedef struct {
    long long x_off, x_start, x_end; /* as fsb_resample_clip: d_x[x_off ..] holds input samples [x_start, x_end) */
    long long j0;       /* first output (absolute index in the row's output) to compute */
    long long out_off;  /* BYTE offset in d_out of output j0, aligned to the format's size */
    long long n_out;    /* outputs computed: j0 .. j0 + n_out - 1 */
    const float* w;     /* as fsb_resample_clip; NULL = no resampling (output j is input j) */
    const int32_t* span;
    long long orig, new_rate;
    long long format;   /* FSB_OUT_* */
} fsb_audio_out_row;

/* Each output y is what fsb_resample computes for it (the same fp64 sum, rounded to fp32 once), stored in the row's
 * format. Rows of different rates and formats share a launch; max_out >= every row's n_out. */
int fsb_audio_out(const float* d_x, const fsb_audio_out_row* d_rows, int B, long long max_out, void* d_out,
                  void* stream);

/* ------------------------------------------------------------------------------------------------
 * Unit-test hooks (used by tests/ only)
 * ---------------------------------------------------------------------------------------------- */
/* out[j][i] (fp32, ld = m) = sum_k A[i][k] * B[j][k]; A [m,k], B [n,k] bf16 row-major, by the prefill / codec GEMM
 * (csrc/gemm_tc.cu). bn in {32,64,128,256}; streamk_ctas > 0 splits the k-blocks over that many CTAs with
 * gemm_plan_streamk and adds the partials in a separate kernel. This is not the decode step GEMM: that one is
 * fsb_op_step_gemm below. */
int fsb_op_gemm(const void* d_a, const void* d_b, float* d_out, int m, int n, int k, int bn,
                int streamk_ctas, void* stream);

/* One decode step GEMM (csrc/lm_gemm.cu) on its own: out[j][i] (fp32, [rows][n_out]) = sum_k W[i][k] * X'[j][k],
 * summed from the stream-K partials in slot order by step_partial_sums, the consumers' own helper (an element where
 * step_partial_sum disagrees with it in any bit is returned as NaN). W bf16 [n_out][K]; X bf16 [32][K], all 32 rows
 * readable; X' = X as given, or, when d_norm_w != NULL, X normalised on load with d_x_ssq (f32 [32][32]: per row, the
 * sums of squares of its 128-feature tiles) and eps. rows in [1, 32]; K a multiple of 8 (<= 4096 with the norm).
 * num_ctas / stages are requests that step_plan_init may clamp; info (host, 5 ints, may be NULL) = CTAs, stages,
 * max partial slots of a tile, max (tile, k-block) units of a CTA, max items (tile ranges) of a CTA of the plan
 * that ran. Synchronises `stream`. */
int fsb_op_step_gemm(const void* d_w, int n_out, int K, const void* d_x, int rows, const void* d_norm_w,
                     const float* d_x_ssq, float eps, int num_ctas, int stages, float* d_out, int* info, void* stream);
/* The same for either row tile of the decode step: row_tile 32 or 64; X bf16 [row_tile][K], all row_tile rows
 * readable; d_x_ssq f32 [row_tile][32]; rows in [1, row_tile]. fsb_op_step_gemm is this with row_tile = 32. */
int fsb_op_step_gemm_tile(const void* d_w, int n_out, int K, const void* d_x, int row_tile, int rows,
                          const void* d_norm_w, const float* d_x_ssq, float eps, int num_ctas, int stages, float* d_out,
                          int* info, void* stream);

/* Runs the step GEMMs of decode layer `layer` of the slow (fast = 0) or fast (fast = 1) stack for `rows` batch rows
 * exactly as fsb_lm_decode does (the handle's own plans, launch order and partial workspace), without attention:
 *   upto = 1: wo GEMM + its residual-add finalize (x += wo(attn) + bo, and the sums of squares of x)
 *   upto = 2: + w1|w3 GEMM (normalised on load) + SwiGLU finalize (h)
 *   upto = 3: + w2 GEMM + its residual-add finalize
 * Inputs and outputs are the fsb_lm_buffer arrays "x_slow" / "x_fast", "ssq_slow" / "ssq_fast", "attn" and "ffn_h".
 * rows in [1, max_batch]. */
int fsb_lm_test_layer_gemms(fsb_lm* h, int fast, int layer, int rows, int upto, void* stream);

/* Runs the qkv step GEMM of decode layer `layer` and the decode attention after it (csrc/lm_kernels.cu
 * attn_decode_kernel: the GEMM's fix-up -- bias, qk-norm, RoPE --, the K/V append and the attention) for `rows` batch
 * rows, with the arguments fsb_lm_decode gives them: the handle's own plan and partial workspace, the "kv_page" table,
 * the context bound (fsb_lm_set_context_bound) and the score chunk (fsb_op_attn_score_chunk); with attn_split set and
 * a bound above it, the slow stack's launch is the split sequence (front end, spans, combine). The GEMM's operand is
 * "x_slow" / "x_fast" exactly as the caller wrote them, normalised on load with "ssq_slow" / "ssq_fast". Row i is
 * slot i at position "pos"[i] in both stacks (decode gives the fast stack its codebook positions instead); -1 parks a
 * row. kv_only != 0 stops after the append, as the fast stack's pass 0 does. Outputs: "attn" (rows at stride H*Dh)
 * and the caches "k_*" / "v_*". rows in [1, max_batch]. */
int fsb_lm_test_layer_attn(fsb_lm* h, int fast, int layer, int rows, int kv_only, void* stream);

/* Runs one stage of slow layer `layer` of the prefill for `rows` token rows exactly as fsb_lm_prefill does (the
 * handle's own plans, the narrow / wide GEMM choice, the "kv_page" table and the context bound), on the fsb_lm_buffer
 * prefill workspaces as the caller left them:
 *   stage 0 (embed; `layer` ignored): d_tokens int32 [rows][C+1] -> "x_prefill", "xn_prefill" (attention_norm of 0)
 *   stage 1 (qkv): qkv GEMM of "xn_prefill" -> "ws_prefill"; bias, qk-norm, RoPE -> "q_prefill" and the K/V of each
 *           row appended at (d_row_seq[i], d_row_pos[i]) through the page table ("k_slow" / "v_slow")
 *   stage 2 (attention): "q_prefill" against the caches -> "attn_prefill" (a row whose history has an unmapped page
 *           reads zeros)
 *   stage 3 (wo): wo GEMM of "attn_prefill" -> "ws_prefill"; "x_prefill" += it + bo; "xn_prefill" = ffn_norm(x)
 *   stage 4 (w1|w3): GEMM of "xn_prefill" -> "ws_prefill"; SwiGLU -> "h_prefill"
 *   stage 5 (w2): w2 GEMM of "h_prefill" -> "ws_prefill"; "x_prefill" += it; "xn_prefill" = the next layer's
 *           attention_norm(x), untouched on the last layer.
 * d_row_seq / d_row_pos int32 [rows] (stages 1 and 2). rows in [1, max(max_rows, 128)]. */
int fsb_lm_test_prefill_stage(fsb_lm* h, int layer, int stage, int rows, const int32_t* d_tokens,
                              const int32_t* d_row_seq, const int32_t* d_row_pos, void* stream);

/* Runs one launch group of a decode frame around its two stacks exactly as fsb_lm_decode (and, for the stages after
 * the slow stack, fsb_lm_prefill's tail) does: the same function, the plans of row tile `tile` (the engine's RT, or 32
 * on an RT = 64 engine), on the fsb_lm_buffer arrays as the caller left them. Row i is slot d_row_slot[i] (NULL: slot i;
 * distinct slots in [0, max_batch), not checked). rows in [1, min(tile, max_batch)].
 *   stage 0 (embed): "cur_tok"[r] -> "x_slow"[r] and "ssq_slow"[r] (row r is slot r; no d_row_slot)
 *   stage 1 (first-frame splice): for each row r whose "first_frame_pending"[r] is set: if "slot_state"[r] is 1 or 3,
 *           "first_frame_x" / "first_frame_ssq"[r] -> "x_slow" / "ssq_slow"[r] and "first_frame_pos"[r] -> "pos"[r];
 *           the flag is cleared in every case (no d_row_slot)
 *   stage 2 (slow head): the head GEMM of "x_slow" normalised on load with "norm" and "ssq_slow", then the slow
 *           sampler -> "cur_tok"[slot][0] (and [1..C] at <|im_end|>), "ras_window", "finished", "slot_state",
 *           "slow_logits" (debug engines); first_frame != 0: the first-frame sampler of fused admission
 *   stage 3 (fast input): norm("x_slow") with "norm" if the model has norm_fastlayer_input (else a copy); with
 *           fast_project_in -> "fast_hidden" (bf16 [RT][dim] at row stride dim), then its GEMM + bias (no residual)
 *           -> "x_fast", "ssq_fast"; without it -> "x_fast", "ssq_fast" directly
 *   stage 4 (fast embed, pass p in [1, C)): fast_embeddings["cur_tok"[slot][p]] -> "x_fast", "ssq_fast"
 *   stage 5 (fast head, pass p in [1, C)): the fast_output GEMM of "x_fast" normalised on load with "fast_norm" and
 *           "ssq_fast", then the codebook sampler -> "cur_tok"[slot][p + 1], "fast_logits"[p - 1] (debug engines)
 *   stage 6 (frame end): for each live slot (any slot without slot control) "cur_tok"[slot] -> "out_tokens" at frame
 *           "n_out"[slot] (not stored at or past max_frames), "n_out" + 1, "pos" + 1 unless the slot freezes at its
 *           limit or <|im_end|> ("slot_state" = 2); then "step" + 1.
 * d_set_pos_rows / d_row_pos_src (int32, both or neither): the prefill tail's arguments -- the head samples without
 * RAS and the frame end sets pos[slot] = d_row_pos_src[d_set_pos_rows[i]] (+ 1 unless frozen); without them the stages
 * take a decode frame's. The sampling stages read `s` (ignored with slot control, may be NULL then). */
int fsb_lm_test_frame_stage(fsb_lm* h, int stage, int tile, int rows, int p, const int32_t* d_row_slot,
                            const int32_t* d_set_pos_rows, const int32_t* d_row_pos_src, int first_frame,
                            const fsb_sampling* s, void* stream);

/* Runs the sampler (csrc/lm_kernels.cu sample_kernel) on its own for `rows` batch rows, with the arguments a decode
 * frame gives it: the slow head's (fast = 0, cb_index = 0; use_ras != 0 as in a decode frame, 0 as in the prefill's) or
 * fast codebook cb_index's (fast = 1, cb_index in [1, num_codebooks), use_ras = 0). d_logits is fp32 [rows][n], n =
 * head_rows (slow) or codebook_size (fast), staged as the single partial of a step GEMM so that the sampler's logit
 * is exactly rbf(d_logits). Row i is slot d_row_slot[i] (NULL: slot i); the slots must lie in [0, max_batch) and be
 * distinct, as in a frame (they are not checked: a slot outside writes outside the state arrays). Everything else is the handle's own state,
 * read and written as a frame does: slot control, "cur_tok", "ras_window", "finished", "slow_logits" / "fast_logits",
 * the noise of fsb_lm_set_sampler_noise and the frame counter "step" (frame counters are not advanced). `s` is
 * ignored with slot control (may be NULL then). rows in [1, max_batch]. Synchronises `stream`. */
int fsb_lm_test_sample(fsb_lm* h, int fast, int cb_index, int rows, const int32_t* d_row_slot, const float* d_logits,
                       int use_ras, const fsb_sampling* s, void* stream);

/* Attention keeps one fp32 score per position and head in shared memory; contexts longer than the buffer are walked
 * in chunks, bit-identically (csrc/lm_kernels.cu attend()).  positions > 0 forces a smaller chunk; 0 = automatic. */
int fsb_op_attn_score_chunk(int positions);
/* fsb_window_attn normally runs the tiled tensor-core kernel (csrc/attn_tile.cu); on != 0 makes it run the per-row
 * kernel, whose attention core is the one of the decode step (what the chunking test above exercises). */
int fsb_op_attn_per_row(int on);

#ifdef __cplusplus
}
#endif
#endif /* FISHB200_H */
