// Memory-bound kernels of the Dual-AR path that are not part of a step GEMM (lm_gemm.cuh):
//   * decode frame: embed, attention over the KV cache, sampling, frame bookkeeping, row gathers / norms that
//     re-seed the residual stream (each leaves the per-128-feature sum of squares the next step GEMM's
//     normalise-on-load needs);
//   * prefill and the codec's WindowLimitedTransformer: consumers of a plain fp32 GEMM result y[row][ld]
//     (residual + fish RMSNorm, q/k/v post-processing, SwiGLU), rounding to bf16 at exactly the points where the
//     reference's bf16 tensors round (llama.py:990-1001 RMSNorm, :891-908 qk-norm/RoPE, :979-987 SwiGLU,
//     :842-845 residual adds).
#pragma once
#include "common.cuh"
#include "lm_gemm.cuh"

namespace fsb {

constexpr int kSsqTile = 128;     // features per sum-of-squares entry (= step GEMM tile)
constexpr int kSsqRowStride = 32; // floats per row (== kSsqStride in lm_gemm.cuh)

struct EmbedArgs {
    const int* tokens;  // [rows][C+1] (row-major per token row)
    const __nv_bfloat16* emb;     // [V, D]
    const __nv_bfloat16* cb_emb;  // [C*cs, D]
    __nv_bfloat16* x;             // [rows, D]
    float* ssq;                   // optional [rows][kSsqRowStride]: sum of x^2 per 128-feature tile
    int rows, D, C, cs, vocab;
    int sem_begin, sem_end;
    int scale;  // scale_codebook_embeddings
};
int launch_embed(const EmbedArgs& a, cudaStream_t st);

// y_out[r] = norm_w ? rbf(rbf(x[src(r)] * rsqrt(mean(x^2) + eps)) * norm_w) : x[src(r)], plus its per-tile sum of squares.
// src(r) = gather ? gather[map(r) * gather_stride] : r   (embedding lookups, last-token rows of a prefill)
struct RowsArgs {
    const __nv_bfloat16* x;     // [*, D]
    const __nv_bfloat16* norm_w;  // [D] or null (plain copy)
    const float* ssq_in;          // [*][kSsqRowStride] per-tile sum of squares of x (required with norm_w)
    __nv_bfloat16* y;           // [rows, D]
    float* ssq;                 // [rows][kSsqRowStride] of y (may be null)
    const int* gather;
    const int* gather_map;
    int gather_stride;
    int rows, D;
    float eps;
};
int launch_rows(const RowsArgs& a, cudaStream_t st);

// x_out = rbf(x_in + rbf(y + bias) [* scale])   (skip the add when y == null)
// n_out = rbf(rbf(x_out * rsqrt(mean(x_out^2)+eps)) * w)     [fish RMSNorm: round, then * weight]
struct ResidNormArgs {
    const float* y;  // [rows][ld] fp32 GEMM result or null
    int ld;
    const __nv_bfloat16* bias;   // [D] or null (attention_o_bias)
    const __nv_bfloat16* scale;  // [D] or null: y *= scale (codec LayerScale, modded_dac.py:329-341)
    const __nv_bfloat16* x_in;   // [rows, D] residual input (null => 0)
    __nv_bfloat16* x_out;        // [rows, D] (may alias x_in; null => don't store)
    const __nv_bfloat16* norm_w;  // [D] (null => no norm output)
    __nv_bfloat16* n_out;         // [rows, D]
    int rows, D;
    float eps;
};
int launch_resid_norm(const ResidNormArgs& a, cudaStream_t st);

// KV cache addressing. kv_page == nullptr: one contiguous block per sequence, [seqs][Hkv][S][Dh] (codec, fast stack).
// Otherwise a pool of pages of kKvPage positions, [n_pages][Hkv][kKvPage][Dh], and position p of sequence b lives in
// page kv_page[b * kv_page_ld + p / kKvPage]; -1 = not mapped, neither read nor written. A page is one K tile of
// attn_tile.cu and a whole number of attend()'s 32-position score chunks, so the paged walk sums the same terms in the
// same order as the contiguous one.
constexpr int kKvPage = 64;
// Element offset of (sequence b, KV head g, position pos) in one layer's cache, or -1 when its page is not mapped.
__device__ __forceinline__ long long kv_offset(const int* kv_page, int kv_page_ld, int b, int g, int pos, int Hkv,
                                               int S, int Dh) {
    if (kv_page == nullptr) return ((static_cast<long long>(b) * Hkv + g) * S + pos) * Dh;
    const int pg = kv_page[static_cast<size_t>(b) * kv_page_ld + pos / kKvPage];
    return pg < 0 ? -1 : ((static_cast<long long>(pg) * Hkv + g) * kKvPage + pos % kKvPage) * Dh;
}
// A third layout, the ring (`ring` != 0 in the argument blocks below; codec streaming, DecodeStreamPool): a contiguous
// block per sequence of S + kKvPage rows, [seqs][Hkv][S + kKvPage][Dh], S a multiple of kKvPage. Position p (any p >= 0)
// lives in row p % S; rows [0, kKvPage) are mirrored in rows [S, S + kKvPage), so that any kKvPage consecutive positions
// are consecutive rows from the row of the first. Only the latest S positions of a sequence are kept: a window
// attention needs S >= window + (positions appended in one call) - 1.
__device__ __forceinline__ long long kv_ring_row(int b, int g, int Hkv, int S) {
    return (static_cast<long long>(b) * Hkv + g) * (S + kKvPage);
}

// q,k,v = rbf(y [+bias]); optional per-head nn.RMSNorm (single rounding); interleaved RoPE in
// fp32 with bf16 tables; q -> qbuf[row][H][Dh]; k,v -> the cache at (row_seq, row_pos) (see kv_offset).
struct QkvPrepArgs {
    const float* y;  // [rows][ld]
    int ld;
    const __nv_bfloat16* bias;  // [(H+2Hkv)*Dh] or null
    const __nv_bfloat16* q_norm;  // [Dh] or null
    const __nv_bfloat16* k_norm;
    const __nv_bfloat16* freqs;  // [S, Dh/2, 2] bf16 (cos, sin)
    const int* row_seq;          // [rows] cache slot of each row
    const int* row_pos;          // [rows] position of each row
    __nv_bfloat16* q;            // [rows, H, Dh]
    __nv_bfloat16* kcache;       // one layer's cache (see kv_offset)
    __nv_bfloat16* vcache;
    const int* kv_page;          // page table or null (contiguous)
    int kv_page_ld;
    int rows, H, Hkv, Dh, S;
    float eps;
    int ring;  // 1: the cache is a ring of S positions (kv_ring_row); head_dim 64 or 128, no page table
};
int launch_qkv_prep(const QkvPrepArgs& a, cudaStream_t st);

// out[row][h][:] = softmax(q.k^T * scale over cache positions [max(0,pos-window+1), pos]) . v
// A row whose history includes an unmapped page attends to nothing: its output row is zero, as for an idle row.
// bf16_math = 1 reproduces the fast-AR hand-rolled attention (llama.py:948-976): scores, scaled
// scores, probabilities and the output are each rounded to bf16.
struct AttnArgs {
    const __nv_bfloat16* q;  // [rows, H, Dh]
    const __nv_bfloat16* kcache;
    const __nv_bfloat16* vcache;
    const int* kv_page;  // page table or null (contiguous, see kv_offset); paged caches take no window
    int kv_page_ld;
    const int* row_seq;
    const int* row_pos;
    __nv_bfloat16* out;  // [rows, H*Dh]
    int rows, H, Hkv, Dh, S;
    int window;  // <=0: unlimited
    int lcap;    // score-buffer length: an upper bound of (row_pos + 1); 0 = cache capacity S
    int bf16_math;
    int ring;    // 1: the cache is a ring of S positions (kv_ring_row); needs 0 < window < S and no page table
};
int launch_attn(const AttnArgs& a, cudaStream_t st);
// csrc/attn_tile.cu: 64 rows of one head per CTA, K/V tiles staged once, mma.sync tensor cores, online softmax; what
// launch_attn uses for >= 64 rows (prefill, codec transformer).
bool attn_tile_supported(const AttnArgs& a);
int launch_attn_tile(const AttnArgs& a, cudaStream_t st);
int attn_init();  // set kernel attributes (idempotent)
void attn_set_score_chunk(int positions);  // tests: force the score-buffer chunk (0 = automatic)
void attn_force_per_row(bool on);          // tests: launch_attn runs the per-row kernel instead of the tiled one

// Decode-step attention: the consumer of the qkv step GEMM. One CTA per (batch row, KV group) first finishes that
// GEMM for its own (G + 2) heads -- slot-ordered sum of the stream-K partials, bias, per-head nn.RMSNorm, interleaved
// RoPE (llama.py:891-908) -- appends K/V to the cache (KVCache.update, llama.py:196-214), then attends over the cache
// with q still in shared memory. kv_only: stop after the append (fast pass 0 of a frame, inference.py:147).
// A row parked at position -1 (idle slot), or whose pages are not all mapped, is skipped.
struct AttnDecodeArgs {
    StepPartials qkv;
    const __nv_bfloat16* bias;    // [(H+2Hkv)*Dh] or null
    const __nv_bfloat16* q_norm;  // [Dh] or null
    const __nv_bfloat16* k_norm;
    const __nv_bfloat16* freqs;   // [S, Dh/2, 2] bf16 (cos, sin)
    __nv_bfloat16* kcache;        // one layer's cache (see kv_offset)
    __nv_bfloat16* vcache;
    const int* kv_page;           // page table or null (contiguous)
    int kv_page_ld;
    const int* row_seq;
    const int* row_pos;
    __nv_bfloat16* out;  // [rows, H*Dh]
    int rows, H, Hkv, Dh, S;
    int lcap;       // score-buffer length: an upper bound of (row_pos + 1); 0 = cache capacity S
    int bf16_math;  // the fast stack's all-bf16 attention (llama.py:948-976)
    int kv_only;
    float eps;
};
// kv_miss: per sequence (row_seq) or null. A row with pos >= 0 that meets an unmapped page stores 1 + pos there if the
// entry is still 0 (the CTA of KV group 0), so that the host learns that the row's attention and the tokens sampled
// from it are void. A kernel argument of its own, not a field of AttnDecodeArgs: the span and combine kernels take
// that struct and do not need it.
int launch_attn_decode(const AttnDecodeArgs& a, cudaStream_t st, int* kv_miss = nullptr);

// The same attention with the history of a LONG row -- more than `span` positions -- split over several CTAs, so that
// one long context does not set the time of the whole launch. Three kernels instead of one:
//   1. attn_decode_split_kernel: attn_decode_kernel's front end and, for rows of at most `span` positions, its
//      attention (the same code, the same bits); for a long row it stores the finished q heads to `q` and stops.
//   2. attn_span_kernel, grid (Hkv, rows, spans): CTA (g, row, s) scores positions [s * span, min(L, (s + 1) * span))
//      of a long row once and stores the span's own maximum, sum of exponentials and unnormalised weighted values
//      (fp32) to `ws`.
//   3. attn_combine_kernel, grid (Hkv, rows): merges a long row's spans in ascending order and rounds to bf16 once.
// Span edges are absolute positions and the merge order is fixed: a long row's bits depend on its own history only,
// not on the slot, the neighbours, `bound` or the number of SMs. They are not the bits of attn_decode_kernel for that
// row (a different summation order), which is why the caller opts in. fp32 attention only (bf16_math == 0).
struct AttnSplit {
    __nv_bfloat16* q;  // [rows, H, Dh] finished q heads of the long rows
    float* ws;         // [rows][Hkv][spans] records of attn_span_floats(G, Dh)
    int span;          // positions per span, a multiple of kKvPage; rows longer than this are split
    int bound;         // upper bound of (row_pos + 1) over the rows: spans = ceil(bound / span) are launched
};
// floats of one span record: acc[G][Dh], then max[G], then sum[G]
constexpr int attn_span_floats(int G, int Dh) { return G * (Dh + 2); }
// the longest span attn_span_kernel can hold in shared memory for this geometry (0: unsupported geometry)
int attn_split_max_span(int H, int Hkv, int Dh);
// a.lcap is the base kernel's score bound as for launch_attn_decode; the caller caps it at sp.span
int launch_attn_decode_split(const AttnDecodeArgs& a, const AttnSplit& sp, cudaStream_t st, int* kv_miss = nullptr);

// h = rbf( rbf(silu(rbf(a))) * rbf(c) ): a = w1 feature i, c = w3 feature i of the fused GEMM result.
// interleaved = 0: a = y[i], c = y[I + i];  1: the step-GEMM row order (w13_gate_row in lm_gemm.cuh)
struct SwigluArgs {
    const float* y;  // [rows][ld]
    int ld;
    __nv_bfloat16* h;  // [rows, I]
    int rows, I;
    int interleaved;
};
int launch_swiglu(const SwigluArgs& a, cudaStream_t st);

// Per-slot request control (continuous batching, SURVEY 8f.1). When `state` is non-null the frame kernels
// take the sampling parameters, the RNG stream and the stop rule from these arrays instead of the per-call
// values, so that every request computes exactly what it would compute alone, whatever shares the batch.
//   state: 0 idle, 1 active, 2 finished (frozen until the host retires it), 3 finishing (set by the slow
//   sampler on <|im_end|>; this frame is still recorded, inference.py:233-234)
struct SlotCtl {
    int* state;
    const int* limit;  // frames this request may produce (the prefill frame included)
    const float* temperature;
    const float* top_p;
    const int* top_k;
    const unsigned long long* seed;
    const int* n_out;  // frames produced so far = RNG counter of the request
};
__device__ __forceinline__ bool slot_live(const SlotCtl& c, int slot) {
    if (c.state == nullptr) return true;
    const int s = c.state[slot];
    return s == 1 || s == 3;
}

constexpr int kSampleMaxN = 8192;  // most candidates the sampler holds (one fp32 logit each in shared memory)

struct SampleArgs {
    StepPartials parts;  // stream-K partials of the (restricted) head GEMM: logit = rbf(slot-ordered sum)
    int n;           // number of candidate entries (<= kSampleMaxN)
    int rows;
    // sampling parameters
    float temperature, top_p;
    int top_k;  // <= 1: rank 0 only (greedy argmax, no RAS re-draw); above 256 the same as 256
    // token mapping for the slow head: entry e -> token id (e < n_sem ? sem_begin + e : im_end_id)
    int slow;  // 1: slow head (RAS + token mapping), 0: fast head (codes)
    int n_sem, sem_begin, im_end_id, codebook_size;
    int use_ras;              // RAS only in decode frames (previous_tokens given)
    int* ras_window;          // [rows][10] ring of previous main tokens (slow only)
    int ras_update;           // push the chosen token into the window
    unsigned long long seed;  // Philox key
    const unsigned long long* rng_offset;  // device counter (frame index) mixed into the stream
    int draw_id;              // distinguishes the samples of one frame
    // outputs
    int* cur_tok;     // [rows][C+1]
    int cb_index;     // slow: writes column 0 (token) and 1 (code a0); fast: writes column cb_index+1
    int num_cb;
    float* logits_out;  // optional [rows][n] fp32 copy of the logits (tests)
    int* finished;      // slow only: set when token == im_end
    const int* row_slot;  // optional: state (cur_tok / window / finished / logits_out) index of a row
    // Test hook (parity with the reference's torch RNG stream): when non-null, draw (frame f, draw d) of
    // slot 0 takes its uniforms U from noise_u[(f * noise_draws + d) * noise_ld + candidate] (the values
    // torch.rand produced in the probs dtype, inference.py:43-46) instead of the Philox stream, and scores
    // are formed in bf16 like the reference's tensors.
    const float* noise_u;
    int noise_draws, noise_ld;
    SlotCtl ctl;
};
int launch_sample(const SampleArgs& a, cudaStream_t st);
// The slow sampler of a decode frame that also serves admitted requests' first frames (fused admission): a row whose
// slot has produced no frame yet (n_out[slot] == 0) samples by the prefill's rule -- no RAS substitution, no
// RAS-window update --, every other row as launch_sample does with a.use_ras / a.ras_update. Slot control only.
int launch_sample_first_frame(const SampleArgs& a, cudaStream_t st);

// Fused admission: a prefill that defers its requests' first frames leaves each sequence's last residual row here, per
// slot, and the next decode frame splices it into its own residual stream right before the head GEMM.
struct FirstFrameArgs {
    __nv_bfloat16* x;          // decode residual stream [RT][D] (stage: rows [0, rows) = the gathered last rows)
    float* ssq;                // its sums of squares [RT][kSsqRowStride]
    __nv_bfloat16* stage_x;    // [max_batch][D] staged last rows, by slot
    float* stage_ssq;          // [max_batch][kSsqRowStride]
    int* stage_pos;            // [max_batch] position of the staged row
    int* pending;              // [max_batch] 1: the slot's first frame is still to run
    int* pos;                  // decode positions [RT]
    const int* slots;          // stage: slot of row i
    const int* last_rows;      // stage: prefill row of sequence i (its position is row_pos[last_rows[i]])
    const int* row_pos;        // stage: positions of the prefill rows
    const int* state;          // splice: slot states (a slot vacated while pending is not spliced)
    int rows, D;
};
// Stage: rows [0, rows) of x / ssq -> their slots' staging rows, with the position of the prefill's last row; the
// slot is marked pending and parked at position -1, so that the frame serving it neither appends K/V for the row nor
// attends for it in the slow stack.
int launch_first_frame_stage(const FirstFrameArgs& a, cudaStream_t st);
// Splice, after the slow stack's last finalize and before the head GEMM: for each of the frame's `rows` rows whose slot
// is pending and live, its staged row and sums of squares replace the frame's row, and its position becomes the staged
// one (frame_end then advances it as the prefill's own frame would); the pending flag is cleared either way.
int launch_first_frame_splice(const FirstFrameArgs& a, cudaStream_t st);

// bookkeeping at the end of a frame for each row's slot:
//   out_tokens[slot][c][n_out[slot]] = cur_tok[slot][c]; n_out[slot]++;
//   pos[slot] = set_pos_rows ? row_pos_src[set_pos_rows[row]] + 1 : pos[slot] + 1;   step++
struct FrameEndArgs {
    const int* cur_tok;
    int* out_tokens;  // [slots][C+1][T_cap]
    int* n_out;
    int* pos;
    const int* row_slot;      // optional
    const int* set_pos_rows;  // optional (prefill): last token row of each sequence
    const int* row_pos_src;
    unsigned long long* step;
    int rows, ncols, T_cap;
    SlotCtl ctl;
};
int launch_frame_end(const FrameEndArgs& a, cudaStream_t st);

// Copy positions [0, n_pos) between pages of a paged cache [layers][n_pages][Hkv][kKvPage][Dh], every layer and KV
// head. Page j of the run is src_tab[j] / dst_tab[j] when the table is given (a slot's row of the page table), else
// src0 + j / dst0 + j. Unmapped or identical pages are skipped.
int launch_kv_copy(__nv_bfloat16* cache, int layers, int n_pages, int Hkv, int Dh, const int* src_tab, int src0,
                   const int* dst_tab, int dst0, int n_pos, cudaStream_t st);

// Everything a decode frame reads back from the previous one for one slot, gathered into / scattered from one blob of
// slot_blob_ints(ncols, T_cap) int32: the slot-control scalars, the frame counter, position, finished flag, RAS window,
// the frame's tokens and the frames produced so far (out_tokens[slot][:, :n_out]). Saving also parks the slot
// (state 0, pos -1: the following frames neither attend for the row nor write its K/V). The slow K/V stays where it
// is, in the pages the slot maps; the fast K/V is rebuilt every frame.
struct SlotStateArgs {
    int *state, *limit;
    float *temperature, *top_p;
    int* top_k;
    unsigned long long* seed;
    int *n_out, *pos, *finished, *ras_window, *cur_tok, *out_tokens;
    int* blob;
    int slot, ncols, T_cap;
};
size_t slot_blob_ints(int ncols, int T_cap);
int launch_slot_save(const SlotStateArgs& a, cudaStream_t st);
int launch_slot_restore(const SlotStateArgs& a, cudaStream_t st);

}  // namespace fsb
