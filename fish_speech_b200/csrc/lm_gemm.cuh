// Step GEMM: the weight-streaming matmul of the Dual-AR decode step (llama.py:831-987 one TransformerBlock;
// inference.py:96-181 one frame).
//
//   D[i][j] = sum_k W[i][k] * X[j][k]        i = output feature (128 per tile: two wgmma of 64 rows)
//                                            j = sequence slot of the batch (< RT, the row tile: 32 or 64)
//
// Life of one launch (one CTA = 5 warps + 4 normaliser warps, two CTAs per SM, the whole grid in one wave):
// The row tile RT is chosen per engine: 32 rows (one wgmma.m64n32k16 per 64 weight rows and k16 step) up to 32
// sequences, 64 rows (the same wgmma issued once per 32-row half of the operand tile, its descriptor 4 KB further)
// up to 64. Every output element sees the same MMA sequence at either tile, so its bits do not depend on RT.
//
//   1. The TMA producer requests the first ring-full of weight tiles at once -- before griddepcontrol.wait, i.e.
//      while the previous kernels are still finishing: weights do not depend on anything.
//   2. Main loop: weights HBM -> shared memory by TMA (SWIZZLE_128B, EVICT_FIRST), operand X by TMA from L2; where X
//      is the residual stream it is *normalised on load* -- four warps apply the reference's RMSNorm
//      (llama.py:990-1001: round(x * rsqrt(mean(x^2) + eps)) * w, two bf16 roundings) in place in shared memory, with
//      the per-row sum of squares the producer of the residual stream left behind -- and wgmma accumulates in
//      registers.  Work is a host-built stream-K schedule: (tile, k-block) units cut into equal contiguous ranges, one per
//      CTA, so every SM streams the same number of weight bytes whatever the shape.
//   3. Each CTA stores its fp32 partials and exits: no tail holds shared memory, so the next GEMM's CTAs move in and
//      start step 1 while this launch drains and its consumer runs.
// Whoever consumes the result finishes the GEMM: it sums the partials IN SLOT ORDER (deterministic, independent of
// arrival order and of the batch) and applies what the reference does next:
//   StepFinalize (this file)   PRO_RESID   bias, residual add, new residual stream + per-128-feature sum of squares
//                                          for the next normalise-on-load                          (llama.py:842-845)
//                              PRO_SWIGLU  silu(w1 x) * w3 x on the row-interleaved w1|w3 result   (llama.py:979-987)
//   attention (lm_kernels.cuh) bias, per-head nn.RMSNorm, RoPE, KV append for the qkv GEMM          (llama.py:891-911)
//   sampler (lm_kernels.cuh)   bf16 logits of the two heads                                        (llama.py:447-457)
// The finish runs in a kernel of its own rather than in a tail of this GEMM (last-arriving CTA) or in the prologue of
// the next GEMM: a tail or a prologue holds the shared memory the next GEMM's weight prefetch needs.
//
// Ordering rule: all step GEMMs of an engine share one partial workspace (step_ws), so a GEMM's single consumer
// (finalize, attention or sampler) must be launched after that GEMM and before the next step GEMM.
#pragma once
#include "gemm_tc.cuh"

namespace fsb {

enum StepPro { PRO_RESID = 1, PRO_SWIGLU = 2 };

constexpr int kStepRows = 32;     // batch rows of the 32-row tile = wgmma N
constexpr int kStepRowsMax = 64;  // the 64-row tile: two wgmma N=32 halves
constexpr int kSsqStride = 32;  // floats per row of a sum-of-squares array: one per 128-feature tile (D <= 4096)

// fp32 stream-K partials of one step GEMM:
//   value(row j, feature i) = sum_{q < nparts[i/128]} ws[((q*tiles + i/128)*rt + j)*128 + i%128]
struct StepPartials {
    const float* ws;
    const int* nparts;  // [tiles]
    int tiles;
    int n_out;      // output features (rows of the weight matrix)
    int max_parts;  // max over tiles of nparts: slots [0, max_parts) exist in ws for every tile
    int rt;         // row tile of the GEMM (32 or 64): rows per (slot, tile) block of ws
};

#ifdef __CUDACC__
// one output element, partials added in slot order
__device__ __forceinline__ float step_partial_sum(const StepPartials& P, int row, int feat) {
    const int tile = feat >> 7;
    const int np = __ldg(P.nparts + tile);
    const float* p = P.ws + (static_cast<size_t>(tile) * P.rt + row) * 128 + (feat & 127);
    const size_t ss = static_cast<size_t>(P.tiles) * P.rt * 128;
    float s = 0.f;
    // The loads are bounded by max_parts (a launch constant), not by this tile's count: they leave together with
    // the load of the count instead of one round trip behind it; slots >= np hold stale data and are not added.
    for (int q = 0; q < P.max_parts; q += 8) {  // eight loads in flight, additions in slot order
        float a[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) a[u] = q + u < P.max_parts ? __ldcg(p + static_cast<size_t>(q + u) * ss) : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u)
            if (q + u < np) s += a[u];
    }
    return s;
}
// N output elements of one row at once: all loads of an 8-slot round are in flight together (N * 8 requests), the
// additions stay in slot order -- bitwise the same sums as step_partial_sum.
template <int N>
__device__ __forceinline__ void step_partial_sums(const StepPartials& P, int row, const int (&feat)[N], const bool (&ok)[N],
                                                  float (&out)[N]) {
    const size_t ss = static_cast<size_t>(P.tiles) * P.rt * 128;
    int np[N];
    const float* p[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
        const int f = ok[k] ? feat[k] : 0;
        np[k] = ok[k] ? __ldg(P.nparts + (f >> 7)) : 0;
        p[k] = P.ws + (static_cast<size_t>(f >> 7) * P.rt + row) * 128 + (f & 127);
        out[k] = 0.f;
    }
    for (int q = 0; q < P.max_parts; q += 8) {  // bounded by the launch constant: see step_partial_sum
        float a[N][8];
#pragma unroll
        for (int k = 0; k < N; ++k)
#pragma unroll
            for (int u = 0; u < 8; ++u)
                a[k][u] = (ok[k] && q + u < P.max_parts) ? __ldcg(p[k] + static_cast<size_t>(q + u) * ss) : 0.f;
#pragma unroll
        for (int k = 0; k < N; ++k)
#pragma unroll
            for (int u = 0; u < 8; ++u)
                if (q + u < np[k]) out[k] += a[k][u];
    }
}
#endif

struct StepGemmParams {
    // ---- schedule ----
    const int4* sched;      // items {tile, kb_begin, kb_end, slot}
    const int* cta_items;   // [grid + 1]
    int tiles, stages;
    int n_out, K;           // output features, reduction length
    int rows;               // live batch rows (<= the row tile RT), set by step_gemm_launch
    unsigned long long a_hint, b_hint;
    float* ws;              // out: [slot][tile][RT rows][128 features] fp32 partials
    // ---- operand X by normalise-on-load (NORM = 1) ----
    const float* x_ssq;           // [RT][kSsqStride] per-tile sum of squares of x
    const __nv_bfloat16* norm_w;  // [K]
    int x_nt;                     // tiles per row in x_ssq
    float eps;
};

// The finish of one step GEMM (`prev`) by step_finalize_kernel, launched right after that GEMM.
struct StepFinalize {
    int pro;                      // PRO_RESID / PRO_SWIGLU
    StepPartials prev;
    const __nv_bfloat16* bias;    // PRO_RESID: [prev.n_out] or null
    const __nv_bfloat16* resid;   // PRO_RESID: [RT][prev.n_out]; may alias x_out; null => no add
    __nv_bfloat16* x_out;         // PRO_RESID: [RT][prev.n_out] new residual stream
    float* ssq_out;               // PRO_RESID: [RT][kSsqStride]
    __nv_bfloat16* h;             // PRO_SWIGLU: [RT][I]; prev tile t = features [64t, 64t+64): lanes 32w+l (l < 16) =
    int I;                        //             w1 row, lanes 32w+16+l = w3 row
    int rows;                     // live batch rows (<= prev.rt), set by step_finalize_launch
};

struct StepGemmPlan {
    CUtensorMap tmA, tmB;
    StepGemmParams p;
    dim3 grid;
    size_t smem;
    int norm;
    int rt;  // row tile: 32 or 64
    void* sched_dev;
    int* cta_items_dev;
    int* nparts_dev;
    int max_parts;
    double weight_bytes;
};

// Operand X = act [row_tile][K] (row_tile 32 or 64), fetched by TMA; norm_on_load: act is the un-normalised residual
// stream (the caller fills p.x_ssq / p.norm_w / p.x_nt / p.eps).
int step_plan_init(StepGemmPlan* plan, const __nv_bfloat16* w, int n_out, int K, const __nv_bfloat16* act,
                   bool norm_on_load, int row_tile, int num_ctas, int stages, float* ws, size_t ws_floats);
// the partials `plan` produces, as a consumer sees them
StepPartials step_plan_partials(const StepGemmPlan& plan);
void step_plan_free(StepGemmPlan* plan);
int step_gemm_launch(const StepGemmPlan& plan, int rows, cudaStream_t stream);  // over `rows` (<= plan.rt) batch rows
// PRO_RESID finish of `src`: x_out = resid + (src + bias) (resid / bias may be null), and its sums of squares
StepFinalize step_finalize_resid(const StepGemmPlan& src, const __nv_bfloat16* bias, const __nv_bfloat16* resid,
                                 __nv_bfloat16* x_out, float* ssq_out);
// PRO_SWIGLU finish of the w1|w3 GEMM `src` into h [RT][I]
StepFinalize step_finalize_swiglu(const StepGemmPlan& src, __nv_bfloat16* h, int I);
int step_finalize_launch(const StepFinalize& fin, int rows, cudaStream_t stream);  // one unit per CTA
int step_gemm_init();  // kernel attributes (idempotent)

// Row index of the fused w1|w3 weight for SwiGLU: h feature f -> row of w1[f]; w3[f] sits 16 rows further.
__host__ __device__ inline int w13_gate_row(int f) { return (f >> 6) * 128 + ((f >> 4) & 3) * 32 + (f & 15); }

}  // namespace fsb
