// Dual-AR engine: owns the KV caches, workspaces and GEMM plans of one model replica and runs
// prefill / per-frame decode as a fixed kernel sequence (captured into a CUDA graph for decode).
//
// HBM layout (all bf16 unless noted)
//   weights            caller-owned, row-major [out, in] as in the checkpoint (TMA-ready, K-major); the fused
//                      w1|w3 matrix has its rows interleaved per 128-row tile (lm_gemm.cuh, w13_gate_row)
//   slow KV cache      [n_layer][kv_pages][Hkv][64][Dh]   x2 (K, V): a pool of 64-position pages; page table "kv_page"
//                      int32 [max_batch][ceil(kv_len / 64)] maps a sequence's positions to pages (-1: not mapped)
//   fast KV cache      [n_fast_layer][max_batch][fHkv][num_codebooks][fDh]  x2
//   decode state       residual streams x_slow / x_fast [RT][D] + their per-128-feature sums of squares
//                      (fp32 [RT][32]); q / attention / SwiGLU operands [RT][*]; logits fp32 [max_batch][n]
//   step_ws            fp32 stream-K partials of the step GEMMs: [slot][tile][RT rows][128 features]
// RT = the decode row tile: 32 for max_batch <= 32 (the 32-row step GEMM), 64 above (the 64-row one). An RT = 64
// engine also holds the 32-row plans of every step GEMM (same weights, same stream-K schedule, the first 32 rows of
// the same operand buffers) and runs a frame of <= 32 rows on them: the same bits in less time.
//   prefill workspaces [max_rows][*] operands + ws fp32 [max_rows][N]
//
// One decode frame (inference.py:96-181) = embed, 36 x {qkv GEMM (norm on load), attention (finishes qkv: bias /
// qk-norm / RoPE / KV append), wo GEMM, finalize (residual add), w1|w3 GEMM (norm on load), finalize (SwiGLU), w2 GEMM,
// finalize (residual add)}, head GEMM + sampler, then 10 fast passes of 4 such layers each: ~640 kernels, eight per
// layer; every GEMM only stores fp32 partials, the kernel launched right after it finishes it (lm_gemm.cuh).
//
// Reference: fish_speech/models/text2semantic/llama.py:390-466 (slow step), :799-817 (fast step),
// fish_speech/models/text2semantic/inference.py:96-181 (one frame), :184-238 (frame loop).
#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/fishb200.h"
#include "gemm_tc.cuh"
#include "lm_gemm.cuh"
#include "lm_kernels.cuh"

using namespace fsb;

namespace {

typedef __nv_bfloat16 bf16;
constexpr int kStepStages = 4;       // ring depth the step GEMM plans start from (step_plan_init may shrink it)

struct LayerW {
    const bf16 *attn_norm, *wqkv, *bqkv, *q_norm, *k_norm, *wo, *bo, *ffn_norm, *w13, *w2;
};
struct StepLayer {
    StepGemmPlan qkv, wo, w13, w2;
    StepFinalize wo_out, w13_out, w2_out;  // residual add (+ bo), SwiGLU, residual add
};
struct PrefillLayer {
    GemmPlan qkv, wo, w13, w2;
    GemmPlan qkv_wide, w13_wide;  // the same GEMMs with 256-row tiles of the token rows (half the weight-tile traffic)
};

struct Stack {
    int D = 0, H = 0, Hkv = 0, Dh = 0, I = 0, nl = 0, S = 0;
    int n13 = 0;  // rows of the interleaved w1|w3 matrix: ceil(I / 64) * 128
    bool qk_norm = false;
    int bf16_math = 0;
    std::vector<LayerW> w;
    std::vector<StepLayer> dec;     // decode: fused step GEMMs at the engine's row tile RT
    std::vector<StepLayer> dec32;   // RT = 64 only: the same GEMMs at the 32-row tile
    std::vector<PrefillLayer> pf;   // prefill: BN=128 tiles, fp32 result + consumer kernels (slow only)
    bf16 *kcache = nullptr, *vcache = nullptr;
    int* kv_page = nullptr;  // slow stack: page table [max_batch][kv_page_ld] of the paged cache; fast stack: contiguous
    int kv_page_ld = 0, n_pages = 0;
    const bf16* freqs = nullptr;
    size_t cache_layer_stride = 0;
    bf16* xres = nullptr;  // decode residual stream [RT][D]
    float* ssq = nullptr;  // its per-tile sums of squares [RT][kSsqStride]
};

// The step GEMM plans one decode frame runs: the engine's RT plans or, on an RT = 64 engine, the 32-row ones.
struct FramePlans {
    int tile;
    const std::vector<StepLayer>* slow;
    const std::vector<StepLayer>* fast;
    const StepGemmPlan *head, *fast_out, *proj;
    const StepFinalize* proj_out;
};

// One captured decode frame and what its capture depended on (fsb_lm_decode's graph cache).
struct DecodeGraph {
    cudaGraphExec_t exec = nullptr;
    int batch = -1, tile = 0, lcap = -1, kernels = 0;
    bool slot_control = false;
    bool first_frame = false;  // fused admission: the splice node and the first-frame sampler
    const float* noise = nullptr;
    fsb_sampling sampling{};
    unsigned long long used = 0;  // last use, for least-recently-used eviction
};
constexpr int kGraphCache = 16;  // captured frames kept per engine

}  // namespace

struct fsb_lm {
    // per-slot request control (continuous batching): see SlotCtl in lm_kernels.cuh
    bool slot_control = false;
    int* slot_state = nullptr;
    int* slot_limit = nullptr;
    float* slot_temperature = nullptr;
    float* slot_top_p = nullptr;
    int* slot_top_k = nullptr;
    unsigned long long* slot_seed = nullptr;
    fsb_lm_config cfg;
    int num_sms = 0;
    int step_ctas = 0;
    int rt = kStepRows;  // decode row tile: 32 or 64 rows (kStepRowsMax) per step GEMM
    Stack slow, fast;
    const bf16 *emb = nullptr, *cb_emb = nullptr, *norm_w = nullptr, *head_w = nullptr;
    const bf16 *fast_emb = nullptr, *fast_norm_w = nullptr, *fast_out_w = nullptr;
    const bf16 *fast_proj_w = nullptr, *fast_proj_b = nullptr;
    int head_rows = 0;
    StepGemmPlan head_plan, fast_out_plan, proj_plan;
    StepFinalize proj_out;  // fast_project_in's bias, no residual add, into the fast residual stream
    StepGemmPlan head_plan32, fast_out_plan32, proj_plan32;  // RT = 64 only: the 32-row plans
    StepFinalize proj_out32;
    int force_tile = 0;      // fsb_lm_set_decode_tile: 0 = by the frame's row count, else 32 or 64
    int last_tile = 0;       // row tile of the last decode frame
    bool has_proj = false;
    // decode workspaces
    bf16 *q_d = nullptr, *attn_d = nullptr, *h_d = nullptr, *hid_d = nullptr;
    float* step_ws = nullptr;
    size_t step_ws_floats = 0;
    float* span_ws = nullptr;  // span records of the split attention (cfg.attn_split > 0), see AttnSplit
    // prefill workspaces
    bf16 *xres_p = nullptr, *xn_p = nullptr, *q_p = nullptr, *attn_p = nullptr, *h_p = nullptr;
    float* ws = nullptr;
    size_t ws_floats = 0;
    // state
    int *cur_tok = nullptr, *out_tokens = nullptr, *n_out = nullptr, *pos = nullptr, *finished = nullptr;
    int *ras_window = nullptr, *iota = nullptr, *fpos = nullptr;
    int* kv_miss = nullptr;  // per slot: 0, or 1 + the position at which decode attention first met an unmapped page
    // fused admission (fsb_lm_prefill_deferred): per slot, the staged last prompt row, its sums of squares and position,
    // and whether its first frame is still to run; the host mirrors the flags (cleared once a frame serving them is
    // enqueued)
    bf16* stage_x = nullptr;
    float* stage_ssq = nullptr;
    int *stage_pos = nullptr, *pending = nullptr;
    std::vector<char> pending_host;
    int n_pending = 0;
    unsigned long long* step = nullptr;
    // debug / test hooks
    float *slow_logits = nullptr, *fast_logits = nullptr;
    const float* noise_u = nullptr;
    int noise_draws = 0, noise_ld = 0;
    int ctx_lcap = 0;  // score-buffer bound for the slow attention (0 = capacity)
    // decode graph cache: one captured frame per (rows, tile, context bound, slot control, noise, sampling)
    std::vector<DecodeGraph> graphs;
    unsigned long long graph_uses = 0;
    long long graph_captures = 0;
    std::vector<void*> owned;
    std::map<std::string, std::pair<void*, size_t>> named;
};

namespace {

template <typename T>
int dalloc(fsb_lm* h, T** p, size_t count, const char* name = nullptr) {
    void* q = nullptr;
    const size_t bytes = std::max<size_t>(count * sizeof(T), 256);
    FSB_CUDA(cudaMalloc(&q, bytes));
    FSB_CUDA(cudaMemset(q, 0, bytes));
    h->owned.push_back(q);
    *p = reinterpret_cast<T*>(q);
    if (name) h->named[name] = {q, count * sizeof(T)};
    return 0;
}

// Prefill plan: A = weight [n_out, k] on the 128 tile rows, B = activations [rows, k], fp32 result ws[row][n_out].
int make_prefill_plan(fsb_lm* h, GemmPlan* plan, const bf16* w, int n_out, int k, const bf16* act, int act_rows,
                      int bn = 128) {
    memset(plan, 0, sizeof(*plan));
    GemmOperand A{w, k, n_out, 1, k, static_cast<long long>(n_out) * k};
    GemmOperand B{act, k, act_rows, 1, k, static_cast<long long>(act_rows) * k};
    GemmParams& p = plan->p;
    p.kb_per_tap = cdiv(k, 64);
    p.num_taps = 1;
    p.a_hint = kEvictNormal;
    p.a_static = 1;
    p.b_hint = kEvictLast;
    p.rows_i = n_out;
    p.mode = 0;
    p.ws = h->ws;
    p.ws_ld = n_out;
    FSB_TRY(gemm_plan_init(plan, A, B, bn, 4, cdiv(n_out, 128), cdiv(act_rows, bn), 1));
    p.rows_j = act_rows;
    p.ws_slot_stride = 0;
    FSB_CHECK(static_cast<size_t>(act_rows) * n_out <= h->ws_floats, "prefill workspace too small");
    return 0;
}

// 256-row tiles once enough token rows exist to fill the SMs with them: per output element the K loop is the same
// sequence of MMAs, so the result does not depend on the tile width (chunked prefill == one pass stays bit-exact)
int launch_rows_of(const GemmPlan& plan, const GemmPlan& wide, int rows, cudaStream_t st);
int launch_rows_of(const GemmPlan& plan, int rows, cudaStream_t st) {
    GemmPlan q = plan;  // restrict the column tiles to the live rows
    q.grid.y = cdiv(rows, plan.bn);
    q.p.rows_j = rows;
    return gemm_launch(q, st);
}

int launch_rows_of(const GemmPlan& plan, const GemmPlan& wide, int rows, cudaStream_t st) {
    static const int sms = [] {
        int d = 0, n = 0;
        cudaGetDevice(&d);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d);
        return n;
    }();
    const long long tiles_wide = static_cast<long long>(wide.grid.x) * cdiv(rows, 256);
    return (rows >= 512 && tiles_wide >= 2 * sms) ? launch_rows_of(wide, rows, st) : launch_rows_of(plan, rows, st);
}

// Step GEMM over the weight `w` [n_out, K]; operand X = act, used as it is. `rt`: the row tile, h->rt or (on an
// RT = 64 engine) 32, whose plan reads the first 32 rows of the same operand buffer.
int make_step_plan(fsb_lm* h, StepGemmPlan* plan, const bf16* w, int n_out, int K, const bf16* act, int rt) {
    return step_plan_init(plan, w, n_out, K, act, false, rt, h->step_ctas, kStepStages, h->step_ws,
                          h->step_ws_floats);
}

// Step GEMM over the weight `w` [n_out, s.D]; operand X = stack s's residual stream, RMSNorm'd with norm_w on load.
int make_norm_step_plan(fsb_lm* h, StepGemmPlan* plan, const bf16* w, int n_out, const Stack& s, const bf16* norm_w,
                        int rt) {
    FSB_TRY(step_plan_init(plan, w, n_out, s.D, s.xres, true, rt, h->step_ctas, kStepStages, h->step_ws,
                           h->step_ws_floats));
    plan->p.x_ssq = s.ssq;
    plan->p.norm_w = norm_w;
    plan->p.x_nt = cdiv(s.D, 128);
    plan->p.eps = h->cfg.norm_eps;
    return 0;
}

// A 32-row plan of an RT = 64 engine must cut its GEMM into the same stream-K ranges as the 64-row plan (the
// schedule is a function of the unit count and the CTA count): then every output element is the same sum of the same
// MMAs at either tile, and a frame's bits do not depend on which tile ran it.
int check_same_schedule(const StepGemmPlan& a, const StepGemmPlan& b) {
    FSB_CHECK(a.grid.x == b.grid.x && a.p.tiles == b.p.tiles && a.p.K == b.p.K && a.max_parts == b.max_parts,
              "fsb_lm_create: the %d- and %d-row step GEMM plans of a %dx%d weight differ in schedule (%u vs %u CTAs, "
              "%d vs %d partial slots)", a.rt, b.rt, a.p.n_out, a.p.K, a.grid.x, b.grid.x, a.max_parts, b.max_parts);
    return 0;
}

FramePlans frame_plans(const fsb_lm* h, int tile) {
    if (tile == h->rt)
        return FramePlans{tile, &h->slow.dec, &h->fast.dec, &h->head_plan, &h->fast_out_plan, &h->proj_plan,
                          &h->proj_out};
    return FramePlans{tile, &h->slow.dec32, &h->fast.dec32, &h->head_plan32, &h->fast_out_plan32, &h->proj_plan32,
                      &h->proj_out32};
}

// The row tile of a decode frame over `batch` rows: the forced one, else 32 where the engine has 32-row plans.
int frame_tile(const fsb_lm* h, int batch) {
    if (h->force_tile != 0) return h->force_tile;
    return (h->rt == kStepRowsMax && batch <= kStepRows) ? kStepRows : h->rt;
}

SlotCtl slot_ctl(const fsb_lm* h) {
    SlotCtl c{};
    if (!h->slot_control) return c;
    c.state = h->slot_state;
    c.limit = h->slot_limit;
    c.temperature = h->slot_temperature;
    c.top_p = h->slot_top_p;
    c.top_k = h->slot_top_k;
    c.seed = h->slot_seed;
    c.n_out = h->n_out;
    return c;
}

// Arguments of layer l's decode attention over `rows` batch rows, the consumer of the qkv GEMM `qkv` ran: one place
// for run_stack_decode and fsb_lm_test_layer_attn, so that the test hook launches exactly what decode launches.
AttnDecodeArgs decode_attn_args(const fsb_lm* h, const Stack& s, int l, const StepGemmPlan& qkv, int rows,
                                const int* row_seq, const int* row_pos, bool kv_only) {
    const LayerW& w = s.w[l];
    AttnDecodeArgs aa{};
    aa.qkv = step_plan_partials(qkv);
    aa.bias = w.bqkv;
    aa.q_norm = s.qk_norm ? w.q_norm : nullptr;
    aa.k_norm = s.qk_norm ? w.k_norm : nullptr;
    aa.freqs = s.freqs;
    aa.kcache = s.kcache + l * s.cache_layer_stride;
    aa.vcache = s.vcache + l * s.cache_layer_stride;
    aa.kv_page = s.kv_page;
    aa.kv_page_ld = s.kv_page_ld;
    aa.row_seq = row_seq;
    aa.row_pos = row_pos;
    aa.out = h->attn_d;
    aa.rows = rows; aa.H = s.H; aa.Hkv = s.Hkv; aa.Dh = s.Dh; aa.S = s.S;
    aa.lcap = (s.bf16_math == 0) ? h->ctx_lcap : 0;  // slow stack: bounded by the live context, not the capacity
    aa.bf16_math = s.bf16_math;
    aa.kv_only = kv_only ? 1 : 0;
    aa.eps = h->cfg.norm_eps;
    return aa;
}

// Layer l's decode attention, the consumer of the qkv GEMM `qkv` ran. With cfg.attn_split set, a slow-stack launch
// whose context bound exceeds it runs as the three kernels of launch_attn_decode_split; the base kernel's score
// buffer then only has to hold the rows that are not split. Every other launch is the single attn_decode_kernel.
int launch_decode_attn(const fsb_lm* h, const Stack& s, int l, const StepGemmPlan& qkv, int rows, const int* row_seq,
                       const int* row_pos, bool kv_only, cudaStream_t st) {
    AttnDecodeArgs aa = decode_attn_args(h, s, l, qkv, rows, row_seq, row_pos, kv_only);
    const int span = h->cfg.attn_split;
    const int bound = h->ctx_lcap > 0 ? h->ctx_lcap : s.S;
    int* kv_miss = s.kv_page ? h->kv_miss : nullptr;  // the paged slow stack only: the fast stack's cache is contiguous
    if (span <= 0 || s.bf16_math != 0 || bound <= span) return launch_attn_decode(aa, st, kv_miss);
    aa.lcap = span;
    return launch_attn_decode_split(aa, AttnSplit{h->q_d, h->span_ws, span, bound}, st, kv_miss);
}

// The first `upto` (GEMM, finalize) pairs of a layer after its attention: wo + residual add, w1|w3 + SwiGLU,
// w2 + residual add.
int run_layer_gemms(const StepLayer& P, int rows, int upto, cudaStream_t st) {
    const StepGemmPlan* gemm[3] = {&P.wo, &P.w13, &P.w2};
    const StepFinalize* fin[3] = {&P.wo_out, &P.w13_out, &P.w2_out};
    for (int k = 0; k < upto; ++k) {
        FSB_TRY(step_gemm_launch(*gemm[k], rows, st));
        FSB_TRY(step_finalize_launch(*fin[k], rows, st));
    }
    return 0;
}

// ---- decode: one transformer stack over the batch rows, eight kernels per layer: qkv GEMM, attention, then the
// three (GEMM, finalize) pairs. ----
int run_stack_decode(fsb_lm* h, Stack& s, const std::vector<StepLayer>& dec, int rows, const int* row_seq,
                     const int* row_pos, bool stop_after_kv, cudaStream_t st) {
    for (int l = 0; l < s.nl; ++l) {
        const StepLayer& P = dec[l];
        FSB_TRY(step_gemm_launch(P.qkv, rows, st));
        const bool kv_only = stop_after_kv && l == s.nl - 1;  // fast pass 0 only fills the KV cache (inference.py:147)
        FSB_TRY(launch_decode_attn(h, s, l, P.qkv, rows, row_seq, row_pos, kv_only, st));
        if (kv_only) return 0;
        FSB_TRY(run_layer_gemms(P, rows, 3, st));
    }
    return 0;
}

EmbedArgs embed_args(fsb_lm* h, const int* tokens, bf16* x, float* ssq, int rows) {
    const fsb_lm_config& c = h->cfg;
    EmbedArgs ea{};
    ea.tokens = tokens;
    ea.emb = h->emb; ea.cb_emb = h->cb_emb; ea.x = x; ea.ssq = ssq;
    ea.rows = rows; ea.D = h->slow.D; ea.C = c.num_codebooks; ea.cs = c.codebook_size; ea.vocab = c.vocab_size;
    ea.sem_begin = c.semantic_begin_id; ea.sem_end = c.semantic_end_id;
    ea.scale = c.scale_codebook_embeddings;
    return ea;
}

// ---- prefill: the same stack over `rows` token rows with wide-N tensor-core GEMMs and consumer kernels. ----
// The stages of one prefill layer, in launch order (fsb_lm_test_prefill_stage runs any one of them).
enum PrefillStage { kPfEmbed = 0, kPfQkv, kPfAttn, kPfWo, kPfW13, kPfW2, kPfStages };

// The prologue: xres_p = embed(tokens), xn_p = attention_norm_0(xres_p).
int prefill_embed(fsb_lm* h, const int* tokens, int rows, cudaStream_t st) {
    Stack& s = h->slow;
    FSB_TRY(launch_embed(embed_args(h, tokens, h->xres_p, nullptr, rows), st));
    ResidNormArgs r{};
    r.x_in = h->xres_p;
    r.norm_w = s.w[0].attn_norm; r.n_out = h->xn_p;
    r.rows = rows; r.D = s.D; r.eps = h->cfg.norm_eps;
    return launch_resid_norm(r, st);
}

// One stage (kPfQkv .. kPfW2) of slow layer l: one place for run_stack_prefill and fsb_lm_test_prefill_stage, so that
// the test hook launches exactly what prefill launches.
int prefill_stage(fsb_lm* h, int l, int stage, int rows, const int* row_seq, const int* row_pos, cudaStream_t st) {
    Stack& s = h->slow;
    const float eps = h->cfg.norm_eps;
    const LayerW& w = s.w[l];
    PrefillLayer& P = s.pf[l];
    switch (stage) {
        case kPfQkv: {
            FSB_TRY(launch_rows_of(P.qkv, P.qkv_wide, rows, st));
            QkvPrepArgs qa{};
            qa.y = h->ws; qa.ld = (s.H + 2 * s.Hkv) * s.Dh;
            qa.bias = w.bqkv;
            qa.q_norm = s.qk_norm ? w.q_norm : nullptr;
            qa.k_norm = s.qk_norm ? w.k_norm : nullptr;
            qa.freqs = s.freqs;
            qa.row_seq = row_seq;
            qa.row_pos = row_pos;
            qa.q = h->q_p;
            qa.kcache = s.kcache + l * s.cache_layer_stride;
            qa.vcache = s.vcache + l * s.cache_layer_stride;
            qa.kv_page = s.kv_page;
            qa.kv_page_ld = s.kv_page_ld;
            qa.rows = rows; qa.H = s.H; qa.Hkv = s.Hkv; qa.Dh = s.Dh; qa.S = s.S;
            qa.eps = eps;
            return launch_qkv_prep(qa, st);
        }
        case kPfAttn: {
            AttnArgs aa{};
            aa.q = h->q_p;
            aa.kcache = s.kcache + l * s.cache_layer_stride;
            aa.vcache = s.vcache + l * s.cache_layer_stride;
            aa.kv_page = s.kv_page;
            aa.kv_page_ld = s.kv_page_ld;
            aa.row_seq = row_seq;
            aa.row_pos = row_pos;
            aa.out = h->attn_p;
            aa.rows = rows; aa.H = s.H; aa.Hkv = s.Hkv; aa.Dh = s.Dh; aa.S = s.S;
            aa.window = 0;
            aa.lcap = h->ctx_lcap;
            aa.bf16_math = 0;
            return launch_attn(aa, st);
        }
        case kPfWo: {
            FSB_TRY(launch_rows_of(P.wo, rows, st));
            ResidNormArgs r1{};
            r1.y = h->ws; r1.ld = s.D;
            r1.bias = w.bo;
            r1.x_in = h->xres_p; r1.x_out = h->xres_p;
            r1.norm_w = w.ffn_norm; r1.n_out = h->xn_p;
            r1.rows = rows; r1.D = s.D; r1.eps = eps;
            return launch_resid_norm(r1, st);
        }
        case kPfW13: {
            FSB_TRY(launch_rows_of(P.w13, P.w13_wide, rows, st));
            SwigluArgs sa{};
            sa.y = h->ws; sa.ld = s.n13;
            sa.h = h->h_p; sa.rows = rows; sa.I = s.I;
            sa.interleaved = 1;
            return launch_swiglu(sa, st);
        }
        case kPfW2: {
            FSB_TRY(launch_rows_of(P.w2, rows, st));
            ResidNormArgs r2{};
            r2.y = h->ws; r2.ld = s.D;
            r2.x_in = h->xres_p; r2.x_out = h->xres_p;
            // the final norm is applied by the head GEMM's normalise-on-load on the last-token rows only
            r2.norm_w = (l + 1 < s.nl) ? s.w[l + 1].attn_norm : nullptr;
            r2.n_out = h->xn_p;
            r2.rows = rows; r2.D = s.D; r2.eps = eps;
            return launch_resid_norm(r2, st);
        }
    }
    set_error("prefill: no stage %d", stage);
    return 1;
}

// On entry xn_p = attention_norm_0(xres_p) (prefill_embed).
int run_stack_prefill(fsb_lm* h, int rows, const int* row_seq, const int* row_pos, cudaStream_t st) {
    for (int l = 0; l < h->slow.nl; ++l)
        for (int stage = kPfQkv; stage < kPfStages; ++stage)
            FSB_TRY(prefill_stage(h, l, stage, rows, row_seq, row_pos, st));
    return 0;
}

// Arguments of the sampler behind the slow head (p = 0) or behind fast pass p's head (codebook p, p >= 1) over `rows`
// batch rows whose logits are `parts`: one place for run_frame_tail and fsb_lm_test_sample, so that the test hook
// launches exactly what a frame launches.
SampleArgs frame_sample_args(const fsb_lm* h, int p, const StepPartials& parts, int rows, const int* row_slot,
                             bool use_ras, const fsb_sampling& sp) {
    const fsb_lm_config& c = h->cfg;
    SampleArgs a{};
    a.ctl = slot_ctl(h);
    a.parts = parts;
    a.rows = rows;
    a.temperature = sp.temperature; a.top_p = sp.top_p; a.top_k = sp.top_k;
    a.seed = sp.seed;
    a.rng_offset = h->step;
    a.cur_tok = h->cur_tok;
    a.num_cb = c.num_codebooks;
    a.row_slot = row_slot;
    a.noise_u = h->noise_u;
    a.noise_draws = h->noise_draws;
    a.noise_ld = h->noise_ld;
    if (p == 0) {
        a.n = h->head_rows;
        a.slow = 1;
        a.n_sem = h->head_rows - 1;
        a.sem_begin = c.semantic_begin_id;
        a.im_end_id = c.im_end_id;
        a.codebook_size = c.codebook_size;
        a.use_ras = use_ras ? 1 : 0;
        a.ras_window = h->ras_window;
        a.ras_update = use_ras ? 1 : 0;
        a.draw_id = 0;
        a.cb_index = 0;
        a.logits_out = h->slow_logits;
        a.finished = h->finished;
    } else {
        a.n = c.codebook_size;
        a.slow = 0;
        a.draw_id = p;
        a.cb_index = p;
        a.logits_out = h->fast_logits ? h->fast_logits + static_cast<size_t>(p - 1) * c.max_batch * c.codebook_size
                                      : nullptr;
    }
    return a;
}

FirstFrameArgs first_frame_args(fsb_lm* h, int rows) {
    FirstFrameArgs a{};
    a.x = h->slow.xres;
    a.ssq = h->slow.ssq;
    a.stage_x = h->stage_x;
    a.stage_ssq = h->stage_ssq;
    a.stage_pos = h->stage_pos;
    a.pending = h->pending;
    a.pos = h->pos;
    a.state = h->slot_state;
    a.rows = rows;
    a.D = h->slow.D;
    return a;
}

// The launches of a decode frame around its two stacks, in launch order (fsb_lm_test_frame_stage runs any one of them):
// embed, [slow stack], first-frame splice, slow head, fast pass 0 input, then per fast pass p: fast embed (p >= 1),
// [fast stack], fast head (p >= 1); frame end.
enum FrameStage { kFrEmbed = 0, kFrSplice, kFrHead, kFrFastIn, kFrFastEmbed, kFrFastHead, kFrEnd, kFrStages };

// What the frame-tail stages of one call share: the frame's rows and the arguments that differ between a decode
// frame and the prefill's tail.
struct FrameRows {
    int rows;
    const int* row_slot;      // row i is slot row_slot[i] (NULL: slot i)
    bool use_ras, first_frame;
    const int* set_pos_rows;  // the prefill's tail: pos[slot] from row_pos_src[set_pos_rows[i]] (NULL: decode)
    const int* row_pos_src;
};

// One stage of a frame on the plans `fp` (fast pass p for kFrFastEmbed / kFrFastHead): one place for decode_one_frame,
// run_frame_tail and fsb_lm_test_frame_stage, so that the test hook launches exactly what a frame launches.
int frame_stage(fsb_lm* h, const FramePlans& fp, int stage, int p, const FrameRows& fr, const fsb_sampling& sp,
                cudaStream_t st) {
    const fsb_lm_config& c = h->cfg;
    const int C = c.num_codebooks;
    const int rows = fr.rows;
    const int* row_slot = fr.row_slot;
    Stack& s = h->slow;
    Stack& f = h->fast;
    switch (stage) {
        case kFrEmbed:  // decode row r is slot r
            return launch_embed(embed_args(h, h->cur_tok, s.xres, s.ssq, rows), st);
        case kFrSplice:
            return launch_first_frame_splice(first_frame_args(h, rows), st);
        case kFrHead: {
            // slow head over the selectable rows (the final norm is applied on load)
            FSB_TRY(step_gemm_launch(*fp.head, rows, st));
            const SampleArgs head_sample =
                frame_sample_args(h, 0, step_plan_partials(*fp.head), rows, row_slot, fr.use_ras, sp);
            return fr.first_frame ? launch_sample_first_frame(head_sample, st) : launch_sample(head_sample, st);
        }
        case kFrFastIn: {
            // fast pass 0 input: hidden = norm(x) (norm_fastlayer_input) [-> fast_project_in]
            // (llama.py:459-461, 819-828)
            RowsArgs hr{};
            hr.x = s.xres;
            hr.ssq_in = s.ssq;
            hr.norm_w = c.norm_fastlayer_input ? h->norm_w : nullptr;
            hr.rows = rows; hr.D = s.D; hr.eps = c.norm_eps;
            if (h->has_proj) {
                hr.y = h->hid_d;
                FSB_TRY(launch_rows(hr, st));
                FSB_TRY(step_gemm_launch(*fp.proj, rows, st));  // fast_project_in
                return step_finalize_launch(*fp.proj_out, rows, st);
            }
            hr.y = f.xres;
            hr.ssq = f.ssq;
            return launch_rows(hr, st);
        }
        case kFrFastEmbed: {
            // input = fast_embeddings[code_{p-1}] ; codes live in cur_tok[slot][p]
            RowsArgs er{};
            er.x = h->fast_emb;
            er.y = f.xres;
            er.ssq = f.ssq;
            er.gather = h->cur_tok + p;
            er.gather_map = row_slot;
            er.gather_stride = C + 1;
            er.rows = rows; er.D = f.D; er.eps = c.norm_eps;
            return launch_rows(er, st);
        }
        case kFrFastHead:
            FSB_TRY(step_gemm_launch(*fp.fast_out, rows, st));
            return launch_sample(frame_sample_args(h, p, step_plan_partials(*fp.fast_out), rows, row_slot, false, sp),
                                 st);
        case kFrEnd: {
            FrameEndArgs fe{};
            fe.ctl = slot_ctl(h);
            fe.cur_tok = h->cur_tok;
            fe.out_tokens = h->out_tokens;
            fe.n_out = h->n_out;
            fe.pos = h->pos;
            fe.row_slot = row_slot;
            fe.set_pos_rows = fr.set_pos_rows;
            fe.row_pos_src = fr.row_pos_src;
            fe.step = h->step;
            fe.rows = rows; fe.ncols = C + 1; fe.T_cap = c.max_frames;
            return launch_frame_end(fe, st);
        }
    }
    set_error("frame: no stage %d", stage);
    return 1;
}

// Head + sampling + fast passes + bookkeeping for `rows` sequences whose last residual-stream rows (un-normed)
// are in slow.xres[0..rows) with their sums of squares in slow.ssq, on the plans `fp`. inference.py:114-181.
int run_frame_tail(fsb_lm* h, const FramePlans& fp, int rows, const int* row_slot, bool use_ras, bool first_frame,
                   const int* set_pos_rows, const int* row_pos_src, const fsb_sampling& sp, cudaStream_t st) {
    const FrameRows fr{rows, row_slot, use_ras, first_frame, set_pos_rows, row_pos_src};
    const int* slots = row_slot ? row_slot : h->iota;
    FSB_TRY(frame_stage(h, fp, kFrHead, 0, fr, sp, st));
    FSB_TRY(frame_stage(h, fp, kFrFastIn, 0, fr, sp, st));
    for (int p = 0; p < h->cfg.num_codebooks; ++p) {
        if (p > 0) FSB_TRY(frame_stage(h, fp, kFrFastEmbed, p, fr, sp, st));
        FSB_TRY(run_stack_decode(h, h->fast, *fp.fast, rows, slots, h->fpos + p * h->rt, p == 0, st));
        if (p > 0) FSB_TRY(frame_stage(h, fp, kFrFastHead, p, fr, sp, st));
    }
    return frame_stage(h, fp, kFrEnd, 0, fr, sp, st);
}

// One frame over rows [0, batch) on the plans of row tile `tile` (batch <= tile). first_frame (fused admission): the
// rows of slots whose first frame a deferred prefill left pending take their staged last prompt row between the slow
// stack and the head, and sample it by the prefill's rule.
int decode_one_frame(fsb_lm* h, int batch, int tile, const fsb_sampling& sp, bool first_frame, cudaStream_t st) {
    const FramePlans fp = frame_plans(h, tile);
    const FrameRows fr{batch, nullptr, true, first_frame, nullptr, nullptr};
    FSB_TRY(frame_stage(h, fp, kFrEmbed, 0, fr, sp, st));
    FSB_TRY(run_stack_decode(h, h->slow, *fp.slow, batch, h->iota, h->pos, false, st));
    if (first_frame) FSB_TRY(frame_stage(h, fp, kFrSplice, 0, fr, sp, st));
    return run_frame_tail(h, fp, batch, nullptr, true, first_frame, nullptr, nullptr, sp, st);
}

// `nframes` frames over rows [0, batch) on row tile `tile`, eagerly or as replays of a captured frame.
int decode_frames(fsb_lm* h, int batch, int tile, int nframes, const fsb_sampling& spr, bool first_frame,
                         int use_graph, cudaStream_t st) {
    const fsb_sampling* sp = &spr;
    if (!use_graph) {
        for (int i = 0; i < nframes; ++i) FSB_TRY(decode_one_frame(h, batch, tile, *sp, first_frame, st));
        return 0;
    }
    DecodeGraph* hit = nullptr;
    for (DecodeGraph& g : h->graphs)
        if (g.batch == batch && g.tile == tile && g.lcap == h->ctx_lcap && g.slot_control == h->slot_control &&
            g.first_frame == first_frame && g.noise == h->noise_u && memcmp(&g.sampling, sp, sizeof(fsb_sampling)) == 0)
            hit = &g;
    if (hit == nullptr) {
        if (static_cast<int>(h->graphs.size()) >= kGraphCache) {  // make room: drop the least recently used frame
            auto lru = std::min_element(h->graphs.begin(), h->graphs.end(),
                                        [](const DecodeGraph& a, const DecodeGraph& b) { return a.used < b.used; });
            cudaGraphExecDestroy(lru->exec);
            h->graphs.erase(lru);
        }
        // capture on a private stream so the caller's stream mode does not matter
        cudaStream_t cs;
        FSB_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
        cudaGraph_t g = nullptr;
        cudaError_t e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
        int rc = 1;
        const int launches_before = g_launch_count;
        if (e == cudaSuccess) {
            rc = decode_one_frame(h, batch, tile, *sp, first_frame, cs);
            e = cudaStreamEndCapture(cs, &g);
        }
        const int kernels = g_launch_count - launches_before;
        g_launch_count = launches_before;  // captured, not launched
        if (e != cudaSuccess || rc != 0 || g == nullptr) {
            if (rc == 0) set_error("decode: graph capture failed: %s", cudaGetErrorString(e));
            cudaStreamDestroy(cs);
            if (g) cudaGraphDestroy(g);
            return 1;
        }
        cudaGraphExec_t ge = nullptr;
        e = cudaGraphInstantiate(&ge, g, 0);
        cudaGraphDestroy(g);
        cudaStreamDestroy(cs);
        if (e != cudaSuccess) {
            set_error("decode: cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
            return 1;
        }
        ++h->graph_captures;
        DecodeGraph d;
        d.exec = ge;
        d.batch = batch;
        d.tile = tile;
        d.lcap = h->ctx_lcap;
        d.kernels = kernels;
        d.slot_control = h->slot_control;
        d.first_frame = first_frame;
        d.noise = h->noise_u;
        d.sampling = *sp;
        h->graphs.push_back(d);
        hit = &h->graphs.back();
    }
    hit->used = ++h->graph_uses;
    for (int i = 0; i < nframes; ++i) {
        FSB_CUDA(cudaGraphLaunch(hit->exec, st));
        g_launch_count += hit->kernels;
    }
    return 0;
}

size_t step_ws_bound(int n_out, int ctas, int rt) {
    const int tiles = cdiv(n_out, 128);
    return static_cast<size_t>(tiles) * (cdiv(ctas, tiles) + 2) * 128 * rt;
}

}  // namespace

extern "C" {

int fsb_lm_create(const fsb_lm_config* cfg, const fsb_lm_weights* w, fsb_lm** out) {
    FSB_CHECK(cfg && w && out, "fsb_lm_create: null argument");
    FSB_CHECK(cfg->max_batch >= 1 && cfg->max_batch <= kStepRowsMax, "max_batch must be in [1,%d]", kStepRowsMax);
    FSB_CHECK(cfg->dim % 8 == 0 && cfg->fast_dim % 8 == 0 && cfg->intermediate % 16 == 0 &&
                  cfg->fast_intermediate % 16 == 0,
              "dims must be multiples of 8, intermediate sizes of 16 (TMA 16-byte strides, SwiGLU interleave)");
    FSB_CHECK(cfg->dim <= 4096 && cfg->fast_dim <= 4096, "model dim above 4096 is not supported");
    FSB_CHECK((cfg->head_dim == 64 || cfg->head_dim == 128) && (cfg->fast_head_dim == 64 || cfg->fast_head_dim == 128),
              "head_dim must be 64 or 128");
    FSB_CHECK(w->head_rows == cfg->semantic_end_id - cfg->semantic_begin_id + 2, "head_rows mismatch");
    // the sampler holds one row's candidates in shared memory: refuse here, not in the middle of the first frame
    FSB_CHECK(w->head_rows >= 1 && w->head_rows <= kSampleMaxN && cfg->codebook_size >= 1 &&
                  cfg->codebook_size <= kSampleMaxN,
              "head_rows=%d and codebook_size=%d must be in [1, %d] (candidates the sampler holds)", w->head_rows,
              cfg->codebook_size, kSampleMaxN);
    FSB_CHECK(cfg->kv_len >= 1 && cfg->kv_pages >= 0, "kv_len must be >= 1 and kv_pages >= 0");
    if (cfg->attn_split != 0) {
        const int most = attn_split_max_span(cfg->n_head, cfg->n_kv_head, cfg->head_dim);
        FSB_CHECK(cfg->attn_split > 0 && cfg->attn_split % kKvPage == 0 && cfg->attn_split <= most,
                  "attn_split=%d must be 0 (off) or a multiple of %d in [%d, %d] (what one span's scores fit in shared "
                  "memory at head_dim %d, %d query heads per KV head)",
                  cfg->attn_split, kKvPage, kKvPage, most, cfg->head_dim,
                  cfg->n_kv_head > 0 ? cfg->n_head / cfg->n_kv_head : 0);
    }
    fsb_lm* h = new fsb_lm();
    h->cfg = *cfg;
    int dev = 0;
    cudaDeviceProp prop;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
        set_error("fsb_lm_create: no CUDA device");
        delete h;
        return 1;
    }
    if (prop.major != 9 || prop.minor != 0) {
        set_error("fishb200 kernels are built for sm_90a only (device is sm_%d%d)", prop.major, prop.minor);
        delete h;
        return 1;
    }
    h->num_sms = prop.multiProcessorCount;
    if (gemm_init() != 0 || attn_init() != 0 || step_gemm_init() != 0) {
        delete h;
        return 1;
    }
    h->step_ctas = h->num_sms * 2;  // two step-GEMM CTAs per SM
    // engines of up to 32 slots keep the 32-row tile; more slots take the 64-row one (same bits per row)
    h->rt = cfg->max_batch <= kStepRows ? kStepRows : kStepRowsMax;
    const int RT = h->rt;

    auto B16 = [](const void* p) { return reinterpret_cast<const bf16*>(p); };
    h->emb = B16(w->d_embeddings);
    h->cb_emb = B16(w->d_codebook_embeddings);
    h->norm_w = B16(w->d_norm);
    h->head_w = B16(w->d_head);
    h->head_rows = w->head_rows;
    h->fast_emb = B16(w->d_fast_embeddings);
    h->fast_norm_w = B16(w->d_fast_norm);
    h->fast_out_w = B16(w->d_fast_output);
    h->fast_proj_w = B16(w->d_fast_proj_w);
    h->fast_proj_b = B16(w->d_fast_proj_b);
    h->has_proj = w->d_fast_proj_w != nullptr;

    Stack& s = h->slow;
    s.D = cfg->dim; s.H = cfg->n_head; s.Hkv = cfg->n_kv_head; s.Dh = cfg->head_dim; s.I = cfg->intermediate;
    s.nl = cfg->n_layer; s.S = cfg->kv_len; s.qk_norm = cfg->qk_norm != 0; s.bf16_math = 0;
    s.n13 = cdiv(s.I, 64) * 128;
    s.freqs = B16(w->d_freqs);
    Stack& f = h->fast;
    f.D = cfg->fast_dim; f.H = cfg->fast_n_head; f.Hkv = cfg->fast_n_kv_head; f.Dh = cfg->fast_head_dim;
    f.I = cfg->fast_intermediate; f.nl = cfg->n_fast_layer; f.S = cfg->num_codebooks;
    f.qk_norm = cfg->fast_qk_norm != 0; f.bf16_math = 1;
    f.n13 = cdiv(f.I, 64) * 128;
    f.freqs = B16(w->d_fast_freqs);
    auto copy_layers = [&](Stack& st, const fsb_lm_layer* L) {
        st.w.resize(st.nl);
        for (int l = 0; l < st.nl; ++l) {
            st.w[l] = LayerW{B16(L[l].d_attn_norm), B16(L[l].d_wqkv), B16(L[l].d_bqkv), B16(L[l].d_q_norm),
                            B16(L[l].d_k_norm), B16(L[l].d_wo), B16(L[l].d_bo), B16(L[l].d_ffn_norm),
                            B16(L[l].d_w13), B16(L[l].d_w2)};
        }
    };
    copy_layers(s, w->layers);
    copy_layers(f, w->fast_layers);

    const int C = cfg->num_codebooks;
    const int Dm = std::max(s.D, f.D), Qm = std::max(s.H * s.Dh, f.H * f.Dh), Im = std::max(s.I, f.I);
    const int Nqkv_s = (s.H + 2 * s.Hkv) * s.Dh, Nqkv_f = (f.H + 2 * f.Hkv) * f.Dh;
    const int R = std::max(cfg->max_rows, 128);
    h->ws_floats = static_cast<size_t>(R) * std::max({Nqkv_s, s.n13, s.D});
    h->step_ws_floats = 0;
    for (int n : {Nqkv_s, Nqkv_f, s.n13, f.n13, s.D, f.D, h->head_rows, cfg->codebook_size})
        h->step_ws_floats = std::max(h->step_ws_floats, step_ws_bound(n, h->step_ctas, RT));
#define TRYC(x)                  \
    do {                         \
        if ((x) != 0) {          \
            fsb_lm_destroy(h);   \
            return 1;            \
        }                        \
    } while (0)
    TRYC(dalloc(h, &h->ws, h->ws_floats, "ws_prefill"));
    TRYC(dalloc(h, &h->step_ws, h->step_ws_floats));
    TRYC(dalloc(h, &s.xres, static_cast<size_t>(RT) * s.D, "x_slow"));
    TRYC(dalloc(h, &s.ssq, static_cast<size_t>(RT) * kSsqStride, "ssq_slow"));
    TRYC(dalloc(h, &f.xres, static_cast<size_t>(RT) * f.D, "x_fast"));
    TRYC(dalloc(h, &f.ssq, static_cast<size_t>(RT) * kSsqStride, "ssq_fast"));
    TRYC(dalloc(h, &h->hid_d, static_cast<size_t>(RT) * Dm, "fast_hidden"));
    TRYC(dalloc(h, &h->q_d, static_cast<size_t>(RT) * Qm, "q"));
    if (cfg->attn_split > 0)
        TRYC(dalloc(h, &h->span_ws,
                    static_cast<size_t>(cfg->max_batch) * s.Hkv * cdiv(cfg->kv_len, cfg->attn_split) *
                        attn_span_floats(s.H / s.Hkv, s.Dh),
                    "attn_span_ws"));
    TRYC(dalloc(h, &h->attn_d, static_cast<size_t>(RT) * Qm, "attn"));
    TRYC(dalloc(h, &h->h_d, static_cast<size_t>(RT) * Im, "ffn_h"));
    TRYC(dalloc(h, &h->xres_p, static_cast<size_t>(R) * s.D, "x_prefill"));
    TRYC(dalloc(h, &h->xn_p, static_cast<size_t>(R) * s.D, "xn_prefill"));
    TRYC(dalloc(h, &h->q_p, static_cast<size_t>(R) * s.H * s.Dh, "q_prefill"));
    TRYC(dalloc(h, &h->attn_p, static_cast<size_t>(R) * s.H * s.Dh, "attn_prefill"));
    TRYC(dalloc(h, &h->h_p, static_cast<size_t>(R) * s.I, "h_prefill"));
    s.kv_page_ld = cdiv(s.S, kKvPage);
    s.n_pages = cfg->kv_pages > 0 ? cfg->kv_pages : cfg->max_batch * s.kv_page_ld;
    s.cache_layer_stride = static_cast<size_t>(s.n_pages) * s.Hkv * kKvPage * s.Dh;
    f.cache_layer_stride = static_cast<size_t>(cfg->max_batch) * f.Hkv * f.S * f.Dh;
    TRYC(dalloc(h, &s.kcache, s.cache_layer_stride * s.nl, "k_slow"));
    TRYC(dalloc(h, &s.vcache, s.cache_layer_stride * s.nl, "v_slow"));
    TRYC(dalloc(h, &f.kcache, f.cache_layer_stride * f.nl, "k_fast"));
    TRYC(dalloc(h, &f.vcache, f.cache_layer_stride * f.nl, "v_fast"));
    TRYC(dalloc(h, &s.kv_page, static_cast<size_t>(cfg->max_batch) * s.kv_page_ld, "kv_page"));
    if (cudaMemset(s.kv_page, 0xff, static_cast<size_t>(cfg->max_batch) * s.kv_page_ld * 4) != cudaSuccess) {
        set_error("fsb_lm_create: page table init failed");  // every entry -1: nothing mapped
        fsb_lm_destroy(h);
        return 1;
    }
    TRYC(dalloc(h, &h->cur_tok, static_cast<size_t>(cfg->max_batch) * (C + 1), "cur_tok"));
    TRYC(dalloc(h, &h->out_tokens, static_cast<size_t>(cfg->max_batch) * (C + 1) * cfg->max_frames, "out_tokens"));
    TRYC(dalloc(h, &h->n_out, cfg->max_batch, "n_out"));
    TRYC(dalloc(h, &h->pos, RT, "pos"));
    TRYC(dalloc(h, &h->finished, cfg->max_batch, "finished"));
    TRYC(dalloc(h, &h->ras_window, static_cast<size_t>(cfg->max_batch) * 10, "ras_window"));
    TRYC(dalloc(h, &h->slot_state, cfg->max_batch, "slot_state"));
    TRYC(dalloc(h, &h->slot_limit, cfg->max_batch, "slot_limit"));
    TRYC(dalloc(h, &h->slot_temperature, cfg->max_batch, "slot_temperature"));
    TRYC(dalloc(h, &h->slot_top_p, cfg->max_batch, "slot_top_p"));
    TRYC(dalloc(h, &h->slot_top_k, cfg->max_batch, "slot_top_k"));
    TRYC(dalloc(h, &h->slot_seed, cfg->max_batch, "slot_seed"));
    TRYC(dalloc(h, &h->kv_miss, cfg->max_batch, "kv_miss"));
    TRYC(dalloc(h, &h->stage_x, static_cast<size_t>(cfg->max_batch) * s.D, "first_frame_x"));
    TRYC(dalloc(h, &h->stage_ssq, static_cast<size_t>(cfg->max_batch) * kSsqStride, "first_frame_ssq"));
    TRYC(dalloc(h, &h->stage_pos, cfg->max_batch, "first_frame_pos"));
    TRYC(dalloc(h, &h->pending, cfg->max_batch, "first_frame_pending"));
    h->pending_host.assign(cfg->max_batch, 0);
    TRYC(dalloc(h, &h->iota, RT));
    TRYC(dalloc(h, &h->fpos, static_cast<size_t>(C) * RT));
    TRYC(dalloc(h, &h->step, 1, "step"));
    if (cfg->debug) {
        TRYC(dalloc(h, &h->slow_logits, static_cast<size_t>(cfg->max_batch) * h->head_rows, "slow_logits"));
        TRYC(dalloc(h, &h->fast_logits, static_cast<size_t>(C) * cfg->max_batch * cfg->codebook_size, "fast_logits"));
    }
    {
        std::vector<int> io(RT), fp(static_cast<size_t>(C) * RT);
        for (int i = 0; i < RT; ++i) io[i] = i;
        for (int p = 0; p < C; ++p)
            for (int i = 0; i < RT; ++i) fp[p * RT + i] = p;
        if (cudaMemcpy(h->iota, io.data(), io.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
            cudaMemcpy(h->fpos, fp.data(), fp.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
            set_error("fsb_lm_create: state upload failed");
            fsb_lm_destroy(h);
            return 1;
        }
    }
    // ---- GEMM plans, and the finalize after each GEMM whose consumer is another GEMM ----
    // the decode plans of one layer at row tile `rt`
    auto build_step = [&](Stack& st, StepLayer& P, const LayerW& lw, int rt) -> int {
        const int Nqkv = (st.H + 2 * st.Hkv) * st.Dh;
        FSB_TRY(make_norm_step_plan(h, &P.qkv, lw.wqkv, Nqkv, st, lw.attn_norm, rt));
        FSB_TRY(make_step_plan(h, &P.wo, lw.wo, st.D, st.H * st.Dh, h->attn_d, rt));
        P.wo_out = step_finalize_resid(P.wo, lw.bo, st.xres, st.xres, st.ssq);
        FSB_TRY(make_norm_step_plan(h, &P.w13, lw.w13, st.n13, st, lw.ffn_norm, rt));
        P.w13_out = step_finalize_swiglu(P.w13, h->h_d, st.I);
        FSB_TRY(make_step_plan(h, &P.w2, lw.w2, st.D, st.I, h->h_d, rt));
        P.w2_out = step_finalize_resid(P.w2, nullptr, st.xres, st.xres, st.ssq);
        return 0;
    };
    const bool two_tiles = RT == kStepRowsMax;
    auto build = [&](Stack& st, bool with_prefill) -> int {
        st.dec.resize(st.nl);
        if (two_tiles) st.dec32.resize(st.nl);
        if (with_prefill) st.pf.resize(st.nl);
        const int Nqkv = (st.H + 2 * st.Hkv) * st.Dh;
        for (int l = 0; l < st.nl; ++l) {
            const LayerW& lw = st.w[l];
            StepLayer& P = st.dec[l];
            FSB_TRY(build_step(st, P, lw, RT));
            if (two_tiles) {
                StepLayer& Q = st.dec32[l];
                FSB_TRY(build_step(st, Q, lw, kStepRows));
                FSB_TRY(check_same_schedule(Q.qkv, P.qkv));
                FSB_TRY(check_same_schedule(Q.wo, P.wo));
                FSB_TRY(check_same_schedule(Q.w13, P.w13));
                FSB_TRY(check_same_schedule(Q.w2, P.w2));
            }
            if (with_prefill) {
                FSB_TRY(make_prefill_plan(h, &st.pf[l].qkv, lw.wqkv, Nqkv, st.D, h->xn_p, R));
                FSB_TRY(make_prefill_plan(h, &st.pf[l].wo, lw.wo, st.D, st.H * st.Dh, h->attn_p, R));
                FSB_TRY(make_prefill_plan(h, &st.pf[l].w13, lw.w13, st.n13, st.D, h->xn_p, R));
                FSB_TRY(make_prefill_plan(h, &st.pf[l].qkv_wide, lw.wqkv, Nqkv, st.D, h->xn_p, R, 256));
                FSB_TRY(make_prefill_plan(h, &st.pf[l].w13_wide, lw.w13, st.n13, st.D, h->xn_p, R, 256));
                FSB_TRY(make_prefill_plan(h, &st.pf[l].w2, lw.w2, st.D, st.I, h->h_p, R));
            }
        }
        return 0;
    };
    TRYC(build(s, true));
    TRYC(build(f, false));
    TRYC(make_norm_step_plan(h, &h->head_plan, h->head_w, h->head_rows, s, h->norm_w, RT));
    TRYC(make_norm_step_plan(h, &h->fast_out_plan, h->fast_out_w, cfg->codebook_size, f, h->fast_norm_w, RT));
    if (h->has_proj) {
        TRYC(make_step_plan(h, &h->proj_plan, h->fast_proj_w, f.D, s.D, h->hid_d, RT));
        h->proj_out = step_finalize_resid(h->proj_plan, h->fast_proj_b, nullptr, f.xres, f.ssq);
    }
    if (two_tiles) {
        TRYC(make_norm_step_plan(h, &h->head_plan32, h->head_w, h->head_rows, s, h->norm_w, kStepRows));
        TRYC(check_same_schedule(h->head_plan32, h->head_plan));
        TRYC(make_norm_step_plan(h, &h->fast_out_plan32, h->fast_out_w, cfg->codebook_size, f, h->fast_norm_w,
                                 kStepRows));
        TRYC(check_same_schedule(h->fast_out_plan32, h->fast_out_plan));
        if (h->has_proj) {
            TRYC(make_step_plan(h, &h->proj_plan32, h->fast_proj_w, f.D, s.D, h->hid_d, kStepRows));
            TRYC(check_same_schedule(h->proj_plan32, h->proj_plan));
            h->proj_out32 = step_finalize_resid(h->proj_plan32, h->fast_proj_b, nullptr, f.xres, f.ssq);
        }
    }
#undef TRYC
    *out = h;
    return 0;
}

void fsb_lm_destroy(fsb_lm* h) {
    if (!h) return;
    for (DecodeGraph& g : h->graphs) cudaGraphExecDestroy(g.exec);
    auto free_plans = [](Stack& st) {
        for (auto& p : st.dec) { step_plan_free(&p.qkv); step_plan_free(&p.wo); step_plan_free(&p.w13); step_plan_free(&p.w2); }
        for (auto& p : st.dec32) { step_plan_free(&p.qkv); step_plan_free(&p.wo); step_plan_free(&p.w13); step_plan_free(&p.w2); }
        for (auto& p : st.pf) { gemm_plan_free(&p.qkv); gemm_plan_free(&p.wo); gemm_plan_free(&p.w13); gemm_plan_free(&p.w2); gemm_plan_free(&p.qkv_wide); gemm_plan_free(&p.w13_wide); }
    };
    free_plans(h->slow);
    free_plans(h->fast);
    step_plan_free(&h->head_plan);
    step_plan_free(&h->fast_out_plan);
    if (h->has_proj) step_plan_free(&h->proj_plan);
    step_plan_free(&h->head_plan32);
    step_plan_free(&h->fast_out_plan32);
    step_plan_free(&h->proj_plan32);
    for (void* p : h->owned) cudaFree(p);
    delete h;
}

int fsb_lm_reset(fsb_lm* h, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const fsb_lm_config& c = h->cfg;
    FSB_CUDA(cudaMemsetAsync(h->n_out, 0, c.max_batch * 4, st));
    FSB_CUDA(cudaMemsetAsync(h->finished, 0, c.max_batch * 4, st));
    FSB_CUDA(cudaMemsetAsync(h->slot_state, 0, c.max_batch * 4, st));
    FSB_CUDA(cudaMemsetAsync(h->ras_window, 0, static_cast<size_t>(c.max_batch) * 10 * 4, st));
    FSB_CUDA(cudaMemsetAsync(h->pos, 0, h->rt * 4, st));
    FSB_CUDA(cudaMemsetAsync(h->step, 0, 8, st));
    FSB_CUDA(cudaMemsetAsync(h->pending, 0, c.max_batch * 4, st));
    std::fill(h->pending_host.begin(), h->pending_host.end(), 0);
    h->n_pending = 0;
    return 0;
}

int fsb_lm_prefill(fsb_lm* h, const int32_t* d_tokens, const int32_t* d_row_slot, const int32_t* d_row_pos,
                   int rows, const int32_t* d_last_rows, const int32_t* d_slots, int nseq, int do_sample,
                   const fsb_sampling* sp, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const fsb_lm_config& c = h->cfg;
    FSB_CHECK(rows >= 1 && rows <= std::max(c.max_rows, 128), "prefill: rows=%d exceeds max_rows=%d", rows, c.max_rows);
    FSB_CHECK(nseq >= 1 && nseq <= c.max_batch, "prefill: nseq=%d out of range", nseq);
    Stack& s = h->slow;
    FSB_TRY(prefill_embed(h, d_tokens, rows, st));
    FSB_TRY(run_stack_prefill(h, rows, d_row_slot, d_row_pos, st));
    if (!do_sample) return 0;
    FSB_CHECK(sp != nullptr || h->slot_control, "prefill: sampling parameters required");
    const fsb_sampling sp_none{1.f, 1.f, 1, 0};
    if (sp == nullptr) sp = &sp_none;
    // last-token rows -> decode residual stream (llama.py:447-448 keeps only the last position)
    RowsArgs g{};
    g.x = h->xres_p;
    g.y = s.xres;
    g.ssq = s.ssq;
    g.gather = d_last_rows;
    g.gather_stride = 1;
    g.rows = nseq; g.D = s.D; g.eps = c.norm_eps;
    FSB_TRY(launch_rows(g, st));
    // the reference resets the RAS window per generate() call and prefill uses no RAS
    return run_frame_tail(h, frame_plans(h, h->rt), nseq, d_slots, false, false, d_last_rows, d_row_pos, *sp, st);
}

int fsb_lm_prefill_deferred(fsb_lm* h, const int32_t* d_tokens, const int32_t* d_row_slot, const int32_t* d_row_pos,
                            int rows, const int32_t* d_last_rows, const int32_t* d_slots, int nseq,
                            const int32_t* h_slots, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(h != nullptr, "prefill_deferred: null handle");
    const fsb_lm_config& c = h->cfg;
    FSB_CHECK(h->slot_control, "prefill_deferred: a deferred first frame needs slot control (fsb_lm_set_slot_control)");
    FSB_CHECK(rows >= 1 && rows <= std::max(c.max_rows, 128), "prefill: rows=%d exceeds max_rows=%d", rows, c.max_rows);
    FSB_CHECK(nseq >= 1 && nseq <= c.max_batch, "prefill: nseq=%d out of range", nseq);
    FSB_CHECK(h_slots != nullptr, "prefill_deferred: null host slot list");
    for (int i = 0; i < nseq; ++i)
        FSB_CHECK(h_slots[i] >= 0 && h_slots[i] < c.max_batch, "prefill_deferred: slot %d outside [0, %d)", h_slots[i],
                  c.max_batch);
    Stack& s = h->slow;
    FSB_TRY(prefill_embed(h, d_tokens, rows, st));
    FSB_TRY(run_stack_prefill(h, rows, d_row_slot, d_row_pos, st));
    // the gather of fsb_lm_prefill's tail, into the same rows; the decode residual stream is free between frames
    RowsArgs g{};
    g.x = h->xres_p;
    g.y = s.xres;
    g.ssq = s.ssq;
    g.gather = d_last_rows;
    g.gather_stride = 1;
    g.rows = nseq; g.D = s.D; g.eps = c.norm_eps;
    FSB_TRY(launch_rows(g, st));
    FirstFrameArgs a = first_frame_args(h, nseq);
    a.slots = d_slots;
    a.last_rows = d_last_rows;
    a.row_pos = d_row_pos;
    FSB_TRY(launch_first_frame_stage(a, st));
    for (int i = 0; i < nseq; ++i) {
        if (!h->pending_host[h_slots[i]]) ++h->n_pending;
        h->pending_host[h_slots[i]] = 1;
    }
    return 0;
}

int fsb_lm_set_slot_control(fsb_lm* h, int enable) {
    FSB_CHECK(h != nullptr, "set_slot_control: null handle");
    h->slot_control = enable != 0;
    return 0;
}

size_t fsb_lm_slot_blob_bytes(fsb_lm* h) {
    if (h == nullptr) return 0;
    return slot_blob_ints(h->cfg.num_codebooks + 1, h->cfg.max_frames) * sizeof(int);
}

// Neither call is part of the decode graph: the graph reads the per-slot arrays at run time, so it stays valid.
static int slot_state_args(fsb_lm* h, int slot, const void* d_blob, const char* what, SlotStateArgs* a) {
    FSB_CHECK(h != nullptr, "%s: null handle", what);
    FSB_CHECK(h->slot_control, "%s: slot control is not enabled (fsb_lm_set_slot_control)", what);
    FSB_CHECK(slot >= 0 && slot < h->cfg.max_batch, "%s: slot=%d outside [0, %d)", what, slot, h->cfg.max_batch);
    FSB_CHECK(d_blob != nullptr, "%s: null blob", what);
    FSB_CHECK((reinterpret_cast<uintptr_t>(d_blob) & 15) == 0, "%s: the blob must be 16-byte aligned", what);
    *a = SlotStateArgs{h->slot_state, h->slot_limit, h->slot_temperature, h->slot_top_p, h->slot_top_k, h->slot_seed,
                       h->n_out, h->pos, h->finished, h->ras_window, h->cur_tok, h->out_tokens,
                       static_cast<int*>(const_cast<void*>(d_blob)), slot, h->cfg.num_codebooks + 1,
                       h->cfg.max_frames};
    return 0;
}

int fsb_lm_slot_save(fsb_lm* h, int slot, void* d_blob, void* stream) {
    SlotStateArgs a{};
    FSB_TRY(slot_state_args(h, slot, d_blob, "slot_save", &a));
    FSB_CHECK(!h->pending_host[slot], "slot_save: slot %d has a deferred first frame that no decode frame has served yet",
              slot);
    return launch_slot_save(a, reinterpret_cast<cudaStream_t>(stream));
}

int fsb_lm_slot_restore(fsb_lm* h, int slot, const void* d_blob, void* stream) {
    SlotStateArgs a{};
    FSB_TRY(slot_state_args(h, slot, d_blob, "slot_restore", &a));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (h->pending_host[slot]) {  // a request vacated before its first frame: the restored one replaces it
        FSB_CUDA(cudaMemsetAsync(h->pending + slot, 0, sizeof(int), st));
        h->pending_host[slot] = 0;
        --h->n_pending;
    }
    return launch_slot_restore(a, st);
}

int fsb_lm_set_sampler_noise(fsb_lm* h, const float* d_u, int draws_per_frame, int ld) {
    FSB_CHECK(h != nullptr, "set_sampler_noise: null handle");
    FSB_CHECK(d_u == nullptr || (draws_per_frame >= 2 * h->cfg.num_codebooks && ld >= h->head_rows && ld >= h->cfg.codebook_size),
              "set_sampler_noise: need >= %d draws per frame and ld >= %d", 2 * h->cfg.num_codebooks,
              std::max(h->head_rows, h->cfg.codebook_size));
    h->noise_u = d_u;
    h->noise_draws = draws_per_frame;
    h->noise_ld = ld;
    return 0;
}

int fsb_lm_decode(fsb_lm* h, int batch, int nframes, const fsb_sampling* sp, int use_graph, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(batch >= 1 && batch <= h->cfg.max_batch, "decode: batch=%d out of range", batch);
    FSB_CHECK(sp != nullptr || h->slot_control, "decode: sampling parameters required");
    const int tile = frame_tile(h, batch);
    FSB_CHECK(batch <= tile, "decode: batch=%d does not fit the forced %d-row tile", batch, tile);
    const fsb_sampling sp_none{1.f, 1.f, 1, 0};
    if (sp == nullptr || h->slot_control) sp = &sp_none;  // per-slot parameters: one graph for every mix of requests
    h->last_tile = tile;
    if (h->n_pending > 0 && nframes >= 1) {
        // fused admission: the first frame also serves the first frames that deferred prefills left pending
        FSB_CHECK(h->slot_control, "decode: slots with a deferred first frame need slot control");
        for (int s = batch; s < h->cfg.max_batch; ++s)
            FSB_CHECK(!h->pending_host[s], "decode: slot %d waits for its first frame outside the batch of %d rows", s,
                      batch);
        FSB_TRY(decode_frames(h, batch, tile, 1, *sp, true, use_graph, st));
        std::fill(h->pending_host.begin(), h->pending_host.end(), 0);
        h->n_pending = 0;
        --nframes;
    }
    return decode_frames(h, batch, tile, nframes, *sp, false, use_graph, st);
}

int fsb_lm_set_decode_tile(fsb_lm* h, int tile) {
    FSB_CHECK(h != nullptr, "set_decode_tile: null handle");
    FSB_CHECK(tile == 0 || tile == kStepRows || tile == kStepRowsMax, "set_decode_tile: tile=%d must be 0, %d or %d",
              tile, kStepRows, kStepRowsMax);
    FSB_CHECK(tile <= h->rt, "set_decode_tile: tile=%d exceeds the engine's %d-row tile (max_batch=%d)", tile, h->rt,
              h->cfg.max_batch);
    h->force_tile = tile;
    return 0;
}

int fsb_lm_decode_tile(fsb_lm* h) { return h ? h->last_tile : 0; }

long long fsb_lm_graph_captures(fsb_lm* h) { return h ? h->graph_captures : 0; }

int fsb_lm_bench_gemms(fsb_lm* h, int reps, double* weight_bytes_per_rep, int* launches_per_rep, void* stream) {
    // Every weight-streaming step GEMM of one decode frame (36 slow layers x 4, head, 10 fast passes x
    // (4 layers x 4 + head)) back to back, without the attention / sampling kernels: the measured stream of the
    // dominant kernel for the roofline line of bench.py. Operands are whatever the workspaces hold; the
    // finalize kernels run (and overwrite the decode state), so call it after the timed generation only.
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const fsb_lm_config& c = h->cfg;
    double bytes = 0;
    int launches = 0;  // GEMMs, not kernels
    const int rows = c.max_batch;
    auto run = [&](const StepGemmPlan& p, const StepFinalize* fin = nullptr) -> int {
        bytes += p.weight_bytes;
        ++launches;
        FSB_TRY(step_gemm_launch(p, rows, st));
        return fin ? step_finalize_launch(*fin, rows, st) : 0;
    };
    for (int r = 0; r < reps; ++r) {
        bytes = 0;
        launches = 0;
        auto stack = [&](Stack& s, bool skip_tail) -> int {
            for (int l = 0; l < s.nl; ++l) {
                FSB_TRY(run(s.dec[l].qkv));
                if (skip_tail && l == s.nl - 1) break;
                FSB_TRY(run(s.dec[l].wo, &s.dec[l].wo_out));
                FSB_TRY(run(s.dec[l].w13, &s.dec[l].w13_out));
                FSB_TRY(run(s.dec[l].w2, &s.dec[l].w2_out));
            }
            return 0;
        };
        FSB_TRY(stack(h->slow, false));
        FSB_TRY(run(h->head_plan));
        for (int p = 0; p < c.num_codebooks; ++p) {
            FSB_TRY(stack(h->fast, p == 0));
            if (p > 0) FSB_TRY(run(h->fast_out_plan));
        }
    }
    if (weight_bytes_per_rep) *weight_bytes_per_rep = bytes;
    if (launches_per_rep) *launches_per_rep = launches;
    return 0;
}

int fsb_lm_bench_step_kind(fsb_lm* h, int kind, int reps, int finalize, double* weight_bytes_per_rep,
                           int* launches_per_rep, void* stream) {
    // The slow stack's step GEMMs of one kind back to back: per kind, the time of a launch against its weight bytes,
    // with and without the finalize kernel in front of it (tools/step_gemm_boundaries.py). Overwrites the decode state.
    FSB_CHECK(h != nullptr, "bench_step_kind: null handle");
    FSB_CHECK(kind >= 0 && kind <= 3, "bench_step_kind: kind=%d outside [0, 3]", kind);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int rows = h->cfg.max_batch;
    double bytes = 0;
    for (int r = 0; r < reps; ++r) {
        bytes = 0;
        for (int l = 0; l < h->slow.nl; ++l) {
            const StepLayer& P = h->slow.dec[l];
            const StepGemmPlan* k[4] = {&P.qkv, &P.wo, &P.w13, &P.w2};
            // what decode runs right before each kind: the finalize of the GEMM that produces its operand
            const StepFinalize* before[4] = {l > 0 ? &h->slow.dec[l - 1].w2_out : nullptr, nullptr, &P.wo_out, &P.w13_out};
            bytes += k[kind]->weight_bytes;
            if (finalize && before[kind]) FSB_TRY(step_finalize_launch(*before[kind], rows, st));
            FSB_TRY(step_gemm_launch(*k[kind], rows, st));
        }
    }
    if (weight_bytes_per_rep) *weight_bytes_per_rep = bytes;
    if (launches_per_rep) *launches_per_rep = h->slow.nl;
    return 0;
}

int fsb_lm_test_layer_gemms(fsb_lm* h, int fast, int layer, int rows, int upto, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(h != nullptr, "test_layer_gemms: null handle");
    Stack& s = fast ? h->fast : h->slow;
    FSB_CHECK(layer >= 0 && layer < s.nl, "test_layer_gemms: layer=%d outside [0, %d)", layer, s.nl);
    FSB_CHECK(rows >= 1 && rows <= h->cfg.max_batch, "test_layer_gemms: rows=%d outside [1, %d]", rows, h->cfg.max_batch);
    FSB_CHECK(upto >= 1 && upto <= 3, "test_layer_gemms: upto=%d outside [1, 3]", upto);
    return run_layer_gemms(s.dec[layer], rows, upto, st);
}

int fsb_lm_test_layer_attn(fsb_lm* h, int fast, int layer, int rows, int kv_only, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(h != nullptr, "test_layer_attn: null handle");
    Stack& s = fast ? h->fast : h->slow;
    FSB_CHECK(layer >= 0 && layer < s.nl, "test_layer_attn: layer=%d outside [0, %d)", layer, s.nl);
    FSB_CHECK(rows >= 1 && rows <= h->cfg.max_batch, "test_layer_attn: rows=%d outside [1, %d]", rows, h->cfg.max_batch);
    // its operand is the residual stream as the caller left it, normalised on load
    const StepGemmPlan& qkv = s.dec[layer].qkv;
    FSB_TRY(step_gemm_launch(qkv, rows, st));
    return launch_decode_attn(h, s, layer, qkv, rows, h->iota, h->pos, kv_only != 0, st);
}

int fsb_lm_test_prefill_stage(fsb_lm* h, int layer, int stage, int rows, const int32_t* d_tokens,
                              const int32_t* d_row_seq, const int32_t* d_row_pos, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(h != nullptr, "test_prefill_stage: null handle");
    const int R = std::max(h->cfg.max_rows, 128);
    FSB_CHECK(stage >= kPfEmbed && stage < kPfStages, "test_prefill_stage: stage=%d outside [0, %d)", stage, kPfStages);
    FSB_CHECK(rows >= 1 && rows <= R, "test_prefill_stage: rows=%d outside [1, %d]", rows, R);
    if (stage == kPfEmbed) {
        FSB_CHECK(d_tokens != nullptr, "test_prefill_stage: the embed stage needs tokens");
        return prefill_embed(h, d_tokens, rows, st);
    }
    FSB_CHECK(layer >= 0 && layer < h->slow.nl, "test_prefill_stage: layer=%d outside [0, %d)", layer, h->slow.nl);
    FSB_CHECK((stage != kPfQkv && stage != kPfAttn) || (d_row_seq != nullptr && d_row_pos != nullptr),
              "test_prefill_stage: stage %d needs the rows' sequences and positions", stage);
    return prefill_stage(h, layer, stage, rows, d_row_seq, d_row_pos, st);
}

int fsb_lm_test_frame_stage(fsb_lm* h, int stage, int tile, int rows, int p, const int32_t* d_row_slot,
                            const int32_t* d_set_pos_rows, const int32_t* d_row_pos_src, int first_frame,
                            const fsb_sampling* sp, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(h != nullptr, "test_frame_stage: null handle");
    const fsb_lm_config& c = h->cfg;
    FSB_CHECK(stage >= kFrEmbed && stage < kFrStages, "test_frame_stage: stage=%d outside [0, %d)", stage, kFrStages);
    FSB_CHECK(tile == h->rt || (tile == kStepRows && h->rt == kStepRowsMax),
              "test_frame_stage: tile=%d is not a row tile of this engine (%d%s)", tile, h->rt,
              h->rt == kStepRowsMax ? " or 32" : "");
    FSB_CHECK(rows >= 1 && rows <= std::min(tile, c.max_batch), "test_frame_stage: rows=%d outside [1, %d]", rows,
              std::min(tile, c.max_batch));
    const bool fast = stage == kFrFastEmbed || stage == kFrFastHead;
    FSB_CHECK(!fast || (p >= 1 && p < c.num_codebooks), "test_frame_stage: p=%d outside [1, %d)", p,
              c.num_codebooks);
    FSB_CHECK((stage != kFrEmbed && stage != kFrSplice) || d_row_slot == nullptr,
              "test_frame_stage: stage %d runs row r as slot r (no row_slot)", stage);
    FSB_CHECK((d_set_pos_rows == nullptr) == (d_row_pos_src == nullptr),
              "test_frame_stage: set_pos_rows and row_pos_src go together");
    FSB_CHECK(!first_frame || (stage == kFrHead && d_set_pos_rows == nullptr),
              "test_frame_stage: first_frame is a decode frame's slow head only");
    FSB_CHECK(sp != nullptr || h->slot_control || (stage != kFrHead && stage != kFrFastHead),
              "test_frame_stage: sampling parameters required");
    const fsb_sampling sp_none{1.f, 1.f, 1, 0};
    // a decode frame's arguments, or the prefill tail's (no RAS) when the positions come from the prefill's rows
    const FrameRows fr{rows, d_row_slot, d_set_pos_rows == nullptr, first_frame != 0, d_set_pos_rows, d_row_pos_src};
    return frame_stage(h, frame_plans(h, tile), stage, fast ? p : 0, fr, (sp && !h->slot_control) ? *sp : sp_none,
                       st);
}

int fsb_lm_test_sample(fsb_lm* h, int fast, int cb_index, int rows, const int32_t* d_row_slot, const float* d_logits,
                       int use_ras, const fsb_sampling* sp, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(h != nullptr, "test_sample: null handle");
    const fsb_lm_config& c = h->cfg;
    FSB_CHECK(rows >= 1 && rows <= c.max_batch, "test_sample: rows=%d outside [1, %d]", rows, c.max_batch);
    FSB_CHECK(fast ? (cb_index >= 1 && cb_index < c.num_codebooks) : cb_index == 0,
              "test_sample: cb_index=%d must be %s", cb_index, fast ? "a sampled codebook in [1, num_codebooks)" : "0");
    FSB_CHECK(!fast || !use_ras, "test_sample: the fast head has no RAS draw");
    FSB_CHECK(d_logits != nullptr, "test_sample: null logits");
    FSB_CHECK(sp != nullptr || h->slot_control, "test_sample: sampling parameters required");
    const fsb_sampling sp_none{1.f, 1.f, 1, 0};
    const int n = fast ? c.codebook_size : h->head_rows;
    // the logits as the single partial of a step GEMM with a row tile of `rows`: ws[tile][row][128]
    const int tiles = cdiv(n, 128);
    const size_t ws_bytes = static_cast<size_t>(tiles) * rows * 128 * sizeof(float);
    float* ws = nullptr;
    int* nparts = nullptr;
    FSB_CUDA(cudaMalloc(&ws, ws_bytes));
    int rc = 1;
    if (cudaMalloc(&nparts, tiles * sizeof(int)) != cudaSuccess) {
        set_error("test_sample: out of device memory");
    } else {
        const std::vector<int> ones(tiles, 1);
        bool ok = cudaMemsetAsync(ws, 0, ws_bytes, st) == cudaSuccess &&
                  cudaMemcpyAsync(nparts, ones.data(), tiles * sizeof(int), cudaMemcpyHostToDevice, st) == cudaSuccess;
        for (int t = 0; ok && t < tiles; ++t)
            ok = cudaMemcpy2DAsync(ws + static_cast<size_t>(t) * rows * 128, 128 * sizeof(float), d_logits + t * 128,
                                   static_cast<size_t>(n) * sizeof(float), std::min(128, n - t * 128) * sizeof(float),
                                   rows, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
        if (!ok) {
            set_error("test_sample: staging the logits failed: %s", cudaGetErrorString(cudaGetLastError()));
        } else {
            const StepPartials P{ws, nparts, tiles, n, 1, rows};
            rc = launch_sample(frame_sample_args(h, fast ? cb_index : 0, P, rows, d_row_slot, use_ras != 0,
                                                 sp ? *sp : sp_none),
                               st);
            const cudaError_t e = cudaStreamSynchronize(st);
            if (rc == 0 && e != cudaSuccess) {
                set_error("test_sample: %s", cudaGetErrorString(e));
                rc = 1;
            }
        }
    }
    cudaFree(nparts);
    cudaFree(ws);
    return rc;
}

int fsb_lm_copy_kv(fsb_lm* h, int src_slot, int dst_slot, int n_pos, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(h != nullptr, "copy_kv: null handle");
    Stack& s = h->slow;
    const int B = h->cfg.max_batch;
    FSB_CHECK(n_pos >= 0 && n_pos <= s.S, "copy_kv: n_pos=%d outside the KV cache (%d)", n_pos, s.S);
    FSB_CHECK(src_slot >= 0 && src_slot < B && dst_slot >= 0 && dst_slot < B, "copy_kv: slot outside [0, %d)", B);
    if (src_slot == dst_slot) return 0;
    const int* src = s.kv_page + static_cast<size_t>(src_slot) * s.kv_page_ld;
    const int* dst = s.kv_page + static_cast<size_t>(dst_slot) * s.kv_page_ld;
    FSB_TRY(launch_kv_copy(s.kcache, s.nl, s.n_pages, s.Hkv, s.Dh, src, 0, dst, 0, n_pos, st));
    FSB_TRY(launch_kv_copy(s.vcache, s.nl, s.n_pages, s.Hkv, s.Dh, src, 0, dst, 0, n_pos, st));
    return 0;
}

int fsb_lm_copy_kv_page(fsb_lm* h, int src_page, int dst_page, int n_pos, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(h != nullptr, "copy_kv_page: null handle");
    Stack& s = h->slow;
    FSB_CHECK(n_pos >= 0 && n_pos <= kKvPage, "copy_kv_page: n_pos=%d outside [0, %d]", n_pos, kKvPage);
    if (src_page == dst_page) return 0;
    FSB_TRY(launch_kv_copy(s.kcache, s.nl, s.n_pages, s.Hkv, s.Dh, nullptr, src_page, nullptr, dst_page, n_pos, st));
    FSB_TRY(launch_kv_copy(s.vcache, s.nl, s.n_pages, s.Hkv, s.Dh, nullptr, src_page, nullptr, dst_page, n_pos, st));
    return 0;
}

int fsb_lm_set_context_bound(fsb_lm* h, int max_positions) {
    // The attention kernel keeps one fp32 score per live position in shared memory; sizing that buffer by
    // the KV capacity would cap max_seq_len at ~12k. The host knows an upper bound of every slot's length
    // (prompt + frames so far): round it up to a 1024 bucket (the decode graph is re-captured per bucket).
    FSB_CHECK(max_positions >= 0, "set_context_bound: negative bound");
    int b = ((max_positions + 1023) / 1024) * 1024;
    if (b > h->cfg.kv_len) b = h->cfg.kv_len;
    h->ctx_lcap = b;
    return 0;
}

int fsb_lm_buffer(fsb_lm* h, const char* name, void** d_ptr, size_t* bytes) {
    auto it = h->named.find(name);
    FSB_CHECK(it != h->named.end(), "fsb_lm_buffer: unknown buffer '%s'", name);
    if (d_ptr) *d_ptr = it->second.first;
    if (bytes) *bytes = it->second.second;
    return 0;
}

}  // extern "C"
