// See lm_gemm.cuh.  CTA = 5 warps (9 when operand X is normalised on load):
//   warps 0-3  one warpgroup: wgmma over the ring, fp32 partial stores of this GEMM from the accumulator registers
//   warp  4    TMA producer (weights and operand X)
//   warps 5-8  operand-X normalisers (NORM == 1): RMSNorm of the TMA-delivered residual rows, in place in the ring
// step_finalize_kernel (the consumer-side finish of a GEMM: residual add / SwiGLU) lives here as well.
#include "lm_gemm.cuh"
#include "wgmma.cuh"

#include <algorithm>
#include <vector>

namespace fsb {

namespace {

// operand-X tile of RT rows (4 KB at 32 rows, 8 KB at 64) and one ring stage (weight tile + operand tile)
template <int RT>
constexpr int kBTileBytesOf = RT * kBlockK * 2;
template <int RT>
constexpr int kStageBytesOf = kATileBytes + kBTileBytesOf<RT>;
constexpr int kHalfBTileBytes = kBTileBytesOf<kStepRows>;  // one 32-row half of the 64-row operand tile
constexpr int kEpiThreads = 128;
constexpr int kMmaThreads = 128;  // one warpgroup
constexpr int kProducerWarp = kMmaThreads / 32;
constexpr int kStepThreads = kMmaThreads + 32;  // + the TMA producer warp
constexpr int kLoaderThreads = 128;  // four normaliser warps: two 16-byte cells per thread and k-block
constexpr int kScratchBytes = 1024;  // r_s[RT] | spare

__device__ __forceinline__ void bar_sync(int id, int n) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// ---- step_finalize: one unit = rows [j0, j0 + R) x the 128 features of tile `tile` of the finished GEMM's output;
// thread tid owns feature tile*128 + tid.  `red` = shared float[4][32]. ----

// Per-row sum over the 128 features of the tile: result for row r in red[q*32 + r], q = 0..3 (one per warp).
template <int R>
__device__ __forceinline__ void rows_warp_sums(const float (&sq)[R], float* red, int quad, int lane) {
    float keep = 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const float s = warp_sum(sq[r]);
        if (lane == r) keep = s;
    }
    red[quad * 32 + lane] = keep;
}

// Slot-ordered sums of the finished GEMM's partials; up to 32 independent loads in flight per thread. RT = the row
// tile of that GEMM (p.prev.rt), a template parameter so that the 32-row finalize keeps its constant strides.
template <int R, int UQ, int RT>  // UQ = partials fetched per round
__device__ __forceinline__ void prev_sums(const StepFinalize& p, int tile, int tid, int j0, float (&acc)[R]) {
    const int np = __ldg(p.prev.nparts + tile);
    const int maxp = p.prev.max_parts;  // loads are bounded by the launch constant, see step_partial_sum
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.f;
    const float* src = p.prev.ws + (static_cast<size_t>(tile) * RT + j0) * 128 + tid;
    const size_t sstride = static_cast<size_t>(p.prev.tiles) * RT * 128;
    for (int q0 = 0; q0 < maxp; q0 += UQ) {
        float t[UQ][R];
#pragma unroll
        for (int u = 0; u < UQ; ++u)
#pragma unroll
            for (int r = 0; r < R; ++r)
                t[u][r] = (q0 + u < maxp && j0 + r < p.rows) ? __ldcg(src + static_cast<size_t>(q0 + u) * sstride + r * 128) : 0.f;
#pragma unroll
        for (int u = 0; u < UQ; ++u) {
            if (q0 + u < np) {
#pragma unroll
                for (int r = 0; r < R; ++r) acc[r] += t[u][r];
            }
        }
    }
}

// llama.py:842-845 / 944-946: y = Linear(...) (bf16), x = x + y (bf16); plus sum_i x^2 of this tile per row
template <int R, int RT>
__device__ __forceinline__ void pro_resid(const StepFinalize& p, int tile, int tid, int j0, float* red) {
    const int quad = tid >> 5, lane = tid & 31;
    const int i = tile * 128 + tid;
    const int n = p.prev.n_out;
    const bool ok = i < n;
    // the loads that do not depend on the partials go first: their round trip overlaps the partial sums
    float xin[R];
#pragma unroll
    for (int r = 0; r < R; ++r)
        xin[r] = (p.resid != nullptr && ok && j0 + r < p.rows) ? bf2f(p.resid[static_cast<size_t>(j0 + r) * n + i]) : 0.f;
    const float b = (p.bias != nullptr && ok) ? bf2f(p.bias[i]) : 0.f;
    float acc[R], sq[R];
    prev_sums<R, 32 / R, RT>(p, tile, tid, j0, acc);
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const float y = p.bias != nullptr ? rbf(acc[r] + b) : rbf(acc[r]);
        const float x = p.resid != nullptr ? rbf(xin[r] + y) : y;
        const bool live = ok && j0 + r < p.rows;
        if (live) p.x_out[static_cast<size_t>(j0 + r) * n + i] = f2bf(x);
        sq[r] = live ? x * x : 0.f;
    }
    rows_warp_sums<R>(sq, red, quad, lane);
    bar_sync(1, kEpiThreads);
    if (quad == 0 && lane < R && j0 + lane < p.rows)
        p.ssq_out[(j0 + lane) * kSsqStride + tile] = ((red[lane] + red[32 + lane]) + red[64 + lane]) + red[96 + lane];
    bar_sync(1, kEpiThreads);
}

// llama.py:979-987: h = silu(w1 x) * w3 x, every intermediate a bf16 tensor
template <int R, int RT>
__device__ __forceinline__ void pro_swiglu(const StepFinalize& p, int tile, int tid, int j0) {
    const int quad = tid >> 5, lane = tid & 31;
    const bool hi = (lane & 16) != 0;  // lanes 16..31 hold the w3 ("up") rows of the features lanes 0..15 gate
    const int f = tile * 64 + quad * 16 + (lane & 15);
    float acc[R];
    prev_sums<R, 32 / R, RT>(p, tile, tid, j0, acc);
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const float up = __shfl_xor_sync(0xffffffffu, acc[r], 16);
        if (!hi && j0 + r < p.rows && f < p.I) {
            const float g = rbf(acc[r]), u = rbf(up);
            const float s = rbf(g / (1.f + expf(-g)));
            p.h[static_cast<size_t>(j0 + r) * p.I + f] = f2bf(s * u);
        }
    }
}

// Batch rows per finalize unit; a load round fetches 32 / R partial slots. PRO_RESID: 4 rows (two rounds for the ~14
// slots of wo / w2 at the engine's schedules) measured faster than 2 or 1 on an H100 SXM. PRO_SWIGLU: 8 rows, one
// round for the <= 4 slots of w1|w3. The sums are added in slot order whatever R is.
template <int PRO>
constexpr int kFinalizeRows = PRO == PRO_SWIGLU ? 8 : 4;

// step_finalize: finishes the GEMM p.prev (one unit = R batch rows x one 128-feature tile per CTA); launched right
// after it, so the next GEMM finds its operand complete.
template <int PRO, int RT>
__global__ void __launch_bounds__(kEpiThreads) step_finalize_kernel(const __grid_constant__ StepFinalize p) {
    constexpr int R = kFinalizeRows<PRO>;
    __shared__ float red[4 * 32];
    pdl_launch_dependents();
    pdl_wait();
    const int units = p.prev.tiles * ((p.rows + R - 1) / R);
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
        const int tile = u % p.prev.tiles, j0 = (u / p.prev.tiles) * R;
        if (PRO == PRO_RESID) pro_resid<R, RT>(p, tile, threadIdx.x, j0, red);
        else pro_swiglu<R, RT>(p, tile, threadIdx.x, j0);
    }
}

template <int NORM, int RT>
__global__ void __launch_bounds__(kStepThreads + (NORM ? kLoaderThreads : 0), 2)
step_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ StepGemmParams p) {
    static_assert(RT == kStepRows || RT == kStepRowsMax, "row tile: 32 or 64");
    constexpr int kStageBytes = kStageBytesOf<RT>;
    constexpr int kBTileBytes = kBTileBytesOf<RT>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t tiles = (raw + 1023u) & ~1023u;  // SWIZZLE_128B tiles need 1024 B alignment
    const int stages = p.stages;
    const uint32_t bars = tiles + static_cast<uint32_t>(stages) * kStageBytes;
    // barrier block: full[stages] (tile ready for the MMA), empty[stages], rawx[stages] (un-normalised X landed)
    const uint32_t full0 = bars, empty0 = bars + 8u * stages, rawx0 = bars + 16u * stages;
    const int scratch_off = ((24 * stages + 15) / 16) * 16;
    uint8_t* gen = smem_raw + (tiles - raw);
    uint8_t* bar_gen = gen + static_cast<size_t>(stages) * kStageBytes;
    float* scratch = reinterpret_cast<float*>(bar_gen + scratch_off);
    float* r_s = scratch;       // [RT] per-row rsqrt (normalisers)
    uint4* normw_s = reinterpret_cast<uint4*>(bar_gen + scratch_off + kScratchBytes);  // [kblocks*8] norm weights

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int item_begin = p.cta_items[blockIdx.x], item_end = p.cta_items[blockIdx.x + 1];

    if (warp == kProducerWarp && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < stages; ++s) {
            mbar_init(full0 + 8u * s, 1 + (NORM ? kLoaderThreads / 32 : 0));
            mbar_init(empty0 + 8u * s, kMmaThreads / 32);  // one arrival per MMA warp
            mbar_init(rawx0 + 8u * s, 1);
        }
        fence_mbar_init();
    }
    __syncthreads();

    pdl_launch_dependents();
    if (warp == kProducerWarp) {
        // ===== TMA producer. Weights do not depend on the upstream kernel: the first ring-full of weight
        // tiles is requested BEFORE griddepcontrol.wait, so this GEMM's HBM stream starts while the previous
        // kernel is still in its tail. Operand X follows once it is complete. =====
        if (lane == 0) {
            int pre = 0;
            {
                int n = item_begin, kb = 0;
                int4 w = make_int4(0, 0, 0, 0);
                if (n < item_end) {
                    w = p.sched[n];
                    kb = w.y;
                }
                while (n < item_end && pre < stages) {
                    const int s = pre;
                    mbar_expect_tx(full0 + 8u * s, NORM ? kATileBytes : kStageBytes);
                    tma_load_3d(tiles + static_cast<uint32_t>(s) * kStageBytes, &tmA, full0 + 8u * s, kb * kBlockK,
                                w.x * kBlockM, 0, p.a_hint);
                    ++pre;
                    if (++kb >= w.z) {
                        if (++n < item_end) {
                            w = p.sched[n];
                            kb = w.y;
                        }
                    }
                }
            }
            pdl_wait();
            int it = 0;
            for (int n = item_begin; n < item_end; ++n) {
                const int4 w = p.sched[n];
                for (int kb = w.y; kb < w.z; ++kb, ++it) {
                    const int s = it % stages;
                    const uint32_t ph = static_cast<uint32_t>(it / stages) & 1u;
                    const uint32_t a_dst = tiles + static_cast<uint32_t>(s) * kStageBytes;
                    if (it >= pre) {
                        mbar_wait(empty0 + 8u * s, ph ^ 1u);
                        mbar_expect_tx(full0 + 8u * s, NORM ? kATileBytes : kStageBytes);
                        tma_load_3d(a_dst, &tmA, full0 + 8u * s, kb * kBlockK, w.x * kBlockM, 0, p.a_hint);
                    }
                    if (NORM) {
                        mbar_expect_tx(rawx0 + 8u * s, kBTileBytes);
                        tma_load_3d(a_dst + kATileBytes, &tmB, rawx0 + 8u * s, kb * kBlockK, 0, 0, p.b_hint);
                    } else {
                        tma_load_3d(a_dst + kATileBytes, &tmB, full0 + 8u * s, kb * kBlockK, 0, 0, p.b_hint);
                    }
                }
            }
        }
    } else if (warp > kProducerWarp) {
        // ===== operand-X normalisers: rbf(rbf(x * r_row) * w) in place on the swizzled tile TMA delivered =====
        if (NORM) {
            const int t = threadIdx.x - kStepThreads;  // 0..127
            // the norm weights are constants: stage them before waiting for the upstream kernel
            const int nchunks = ((p.K + kBlockK - 1) / kBlockK) * 8;
            for (int ch = t; ch < nchunks; ch += kLoaderThreads)
                normw_s[ch] = ch * 8 < p.K ? __ldg(reinterpret_cast<const uint4*>(p.norm_w + ch * 8)) : make_uint4(0, 0, 0, 0);
            pdl_wait();
            if (t < RT) {
                // rsqrt(mean(x^2) + eps) of row t: the producer's per-tile sums, added in tile order (all loads in flight)
                // (16-byte loads: every CTA of the grid reads these same RT lines right after the grid-wide arrival)
                const float4* q = reinterpret_cast<const float4*>(p.x_ssq + t * kSsqStride);
                float4 a[kSsqStride / 4];
#pragma unroll
                for (int u = 0; u < kSsqStride / 4; ++u) a[u] = 4 * u < p.x_nt ? __ldcg(q + u) : make_float4(0.f, 0.f, 0.f, 0.f);
                float tot = 0.f;
#pragma unroll
                for (int u = 0; u < kSsqStride / 4; ++u) {
                    if (4 * u < p.x_nt) tot += a[u].x;
                    if (4 * u + 1 < p.x_nt) tot += a[u].y;
                    if (4 * u + 2 < p.x_nt) tot += a[u].z;
                    if (4 * u + 3 < p.x_nt) tot += a[u].w;
                }
                r_s[t] = rsqrtf(tot / static_cast<float>(p.K) + p.eps);
            }
            bar_sync(2, kLoaderThreads);
            // RT rows x 8 sixteen-byte chunks per k-block; thread t owns chunk (t & 7) of rows (t >> 3) + 16e
            constexpr int kCells = RT * 8 / kLoaderThreads;
            const int c = t & 7, rb = t >> 3;
            float rr[kCells];
            uint32_t off[kCells];
#pragma unroll
            for (int e = 0; e < kCells; ++e) {
                const int row = rb + (kLoaderThreads / 8) * e;
                rr[e] = r_s[row];
                off[e] = static_cast<uint32_t>(row * 128 + ((c ^ (row & 7)) << 4));  // SWIZZLE_128B
            }
            int it = 0;
            for (int n = item_begin; n < item_end; ++n) {
                const int4 w = p.sched[n];
                for (int kb = w.y; kb < w.z; ++kb, ++it) {
                    const int s = it % stages;
                    const uint32_t ph = static_cast<uint32_t>(it / stages) & 1u;
                    const uint4 wv = normw_s[kb * 8 + c];
                    const float wf[8] = {bf_lo(wv.x), bf_hi(wv.x), bf_lo(wv.y), bf_hi(wv.y),
                                         bf_lo(wv.z), bf_hi(wv.z), bf_lo(wv.w), bf_hi(wv.w)};
                    uint8_t* btile = gen + static_cast<size_t>(s) * kStageBytes + kATileBytes;
                    mbar_wait(rawx0 + 8u * s, ph);
#pragma unroll
                    for (int e = 0; e < kCells; ++e) {
                        uint4* cell = reinterpret_cast<uint4*>(btile + off[e]);
                        const uint4 xv = *cell;
                        const float xf[8] = {bf_lo(xv.x), bf_hi(xv.x), bf_lo(xv.y), bf_hi(xv.y),
                                             bf_lo(xv.z), bf_hi(xv.z), bf_lo(xv.w), bf_hi(xv.w)};
                        float nf[8];
#pragma unroll
                        for (int q = 0; q < 8; ++q) nf[q] = rbf(rbf(xf[q] * rr[e]) * wf[q]);
                        uint4 o;
                        o.x = pack_bf2(nf[0], nf[1]);
                        o.y = pack_bf2(nf[2], nf[3]);
                        o.z = pack_bf2(nf[4], nf[5]);
                        o.w = pack_bf2(nf[6], nf[7]);
                        *cell = o;
                    }
                    fence_proxy_async();  // generic-proxy stores -> visible to the tensor core's async proxy
                    __syncwarp();
                    if (lane == 0) mbar_arrive(full0 + 8u * s);
                }
            }
        }
    } else {
        // ===== warpgroup 0: wgmma over the ring (rows [0, 64) and [64, 128) of the weight tile; at RT = 64 each once
        // per 32-row half of the operand tile, with the wgmma of the 32-row tile), then the fp32 partial stores
        // straight from the accumulator registers =====
        pdl_wait();
        int it = 0;
        for (int n = item_begin; n < item_end; ++n) {
            const int4 w = p.sched[n];
            const int tile = w.x, slot = w.w;
            // d0 / d1: weight rows [0, 64) / [64, 128); entries [16h, 16h + 16) hold operand rows [32h, 32h + 32)
            float d0[RT / 2], d1[RT / 2];
#pragma unroll
            for (int e = 0; e < RT / 2; ++e) d0[e] = d1[e] = 0.f;
            for (int kb = w.y; kb < w.z; ++kb, ++it) {
                const int s = it % stages;
                mbar_wait(full0 + 8u * s, static_cast<uint32_t>(it / stages) & 1u);
                const uint32_t a_src = tiles + static_cast<uint32_t>(s) * kStageBytes;
                const uint64_t a0 = make_gdesc(a_src), a1 = make_gdesc(a_src + kHalfATileBytes);
                const uint64_t bd = make_gdesc(a_src + kATileBytes);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kBlockK / 16; ++k) {
#pragma unroll
                    for (int hh = 0; hh < RT / kStepRows; ++hh) {
                        const uint64_t bh = hh == 0 ? bd : make_gdesc(a_src + kATileBytes + hh * kHalfBTileBytes);
                        wgmma_bf16<kStepRows>(d0 + 16 * hh, a0 + 2u * k, bh + 2u * k, 1);
                        wgmma_bf16<kStepRows>(d1 + 16 * hh, a1 + 2u * k, bh + 2u * k, 1);
                    }
                }
                wgmma_commit();
                // release the slot as soon as its own MMAs retire: the producer refills it while the next k-block
                // is multiplied, so the whole ring depth stays in flight
                wgmma_wait<0>();
                __syncwarp();
                if (lane == 0) mbar_arrive(empty0 + 8u * s);
            }
            // accumulator element (feature i, batch row j) -> ws[slot][tile][j][i]
            float* dst = p.ws + ((static_cast<size_t>(slot) * p.tiles + tile) * RT) * 128;
            const int i0 = warp * 16 + (lane >> 2);
#pragma unroll
            for (int b = 0; b < RT / 8; ++b)
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int j = 8 * b + 2 * (lane & 3) + (r & 1);
                    const int i = i0 + 8 * (r >> 1);
                    if (j < p.rows) {
                        __stcg(dst + j * 128 + i, d0[4 * b + r]);
                        __stcg(dst + j * 128 + 64 + i, d1[4 * b + r]);
                    }
                }
        }
    }
}

template <int NORM, int RT>
int launch_t(const StepGemmPlan& plan, const StepGemmParams& p, cudaStream_t st) {
    auto k = step_gemm_kernel<NORM, RT>;
    FSB_LAUNCH(k, plan.grid, dim3(kStepThreads + (NORM ? kLoaderThreads : 0)), plan.smem, st, plan.tmA, plan.tmB, p);
    return 0;
}

const void* kernel_of(int norm, int rt) {
    if (rt == kStepRowsMax)
        return norm ? reinterpret_cast<const void*>(step_gemm_kernel<1, kStepRowsMax>)
                    : reinterpret_cast<const void*>(step_gemm_kernel<0, kStepRowsMax>);
    return norm ? reinterpret_cast<const void*>(step_gemm_kernel<1, kStepRows>)
                : reinterpret_cast<const void*>(step_gemm_kernel<0, kStepRows>);
}

}  // namespace

int step_gemm_init() {
    static bool done = false;
    if (done) return 0;
#define FSB_STEP_ATTR(B_, RT_)                                                                                          \
    FSB_CUDA(cudaFuncSetAttribute(step_gemm_kernel<B_, RT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); \
    FSB_CUDA(cudaFuncSetAttribute(step_gemm_kernel<B_, RT_>, cudaFuncAttributePreferredSharedMemoryCarveout,            \
                                  cudaSharedmemCarveoutMaxShared));
    FSB_STEP_ATTR(1, kStepRows) FSB_STEP_ATTR(0, kStepRows) FSB_STEP_ATTR(1, kStepRowsMax) FSB_STEP_ATTR(0, kStepRowsMax)
#undef FSB_STEP_ATTR
    done = true;
    return 0;
}

int step_plan_init(StepGemmPlan* plan, const __nv_bfloat16* w, int n_out, int K, const __nv_bfloat16* act,
                   bool norm_on_load, int row_tile, int num_ctas, int stages, float* ws, size_t ws_floats) {
    memset(plan, 0, sizeof(*plan));
    FSB_CHECK(K % 8 == 0, "step GEMM: K=%d must be a multiple of 8", K);
    FSB_CHECK(act != nullptr, "step GEMM: operand X missing");
    FSB_CHECK(row_tile == kStepRows || row_tile == kStepRowsMax, "step GEMM: row tile %d is not %d or %d", row_tile,
              kStepRows, kStepRowsMax);
    const int norm = norm_on_load ? 1 : 0;
    const void* kernel = kernel_of(norm, row_tile);
    FSB_TRY(step_gemm_init());
    GemmOperand A{w, K, n_out, 1, K, static_cast<long long>(n_out) * K};
    FSB_TRY(gemm_make_tmap(&plan->tmA, A, kBlockM));
    GemmOperand B{act, K, row_tile, 1, K, static_cast<long long>(row_tile) * K};
    FSB_TRY(gemm_make_tmap(&plan->tmB, B, row_tile));
    const int tiles = cdiv(n_out, kBlockM), kblocks = cdiv(K, kBlockK);
    const int normw_bytes = norm ? kblocks * 128 : 0;
    const size_t stage_bytes = row_tile == kStepRowsMax ? kStageBytesOf<kStepRowsMax> : kStageBytesOf<kStepRows>;
    auto smem_of = [&](int st) {
        return static_cast<size_t>(1024) + static_cast<size_t>(st) * stage_bytes + ((24 * st + 15) / 16) * 16 +
               kScratchBytes + normw_bytes;
    };
    while (stages > 2 && 2 * (smem_of(stages) + 1024) > 228 * 1024) --stages;  // two CTAs per SM
    FSB_CHECK(stages >= 2, "step GEMM: ring too shallow");
    // One wave: the stream-K ranges assume every CTA runs at once.
    int dev = 0, sms = 0, per_sm = 0;
    FSB_CUDA(cudaGetDevice(&dev));
    FSB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    FSB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kStepThreads + (norm ? kLoaderThreads : 0),
                                                           smem_of(stages)));
    FSB_CHECK(per_sm >= 1, "step GEMM: kernel does not fit an SM (smem %zu)", smem_of(stages));
    if (num_ctas > per_sm * sms) num_ctas = per_sm * sms;
    // stream-K: units are (tile, k-block) pairs in tile-major order; CTA c streams units [c*U/n, (c+1)*U/n)
    const long long U = static_cast<long long>(tiles) * kblocks;
    if (num_ctas > U) num_ctas = static_cast<int>(U);
    std::vector<int4> items;
    std::vector<int> cta_items(num_ctas + 1, 0), nparts(tiles, 0);
    for (int c = 0; c < num_ctas; ++c) {
        long long u0 = U * c / num_ctas;
        const long long u1 = U * (c + 1) / num_ctas;
        cta_items[c] = static_cast<int>(items.size());
        while (u0 < u1) {
            const int t = static_cast<int>(u0 / kblocks);
            const long long tend = static_cast<long long>(t + 1) * kblocks;
            const long long e = u1 < tend ? u1 : tend;
            items.push_back(make_int4(t, static_cast<int>(u0 - static_cast<long long>(t) * kblocks),
                                      static_cast<int>(e - static_cast<long long>(t) * kblocks), nparts[t]++));
            u0 = e;
        }
    }
    cta_items[num_ctas] = static_cast<int>(items.size());
    int maxp = 0;
    for (int t = 0; t < tiles; ++t) maxp = std::max(maxp, nparts[t]);
    plan->max_parts = maxp;
    FSB_CHECK(static_cast<size_t>(maxp) * tiles * 128 * row_tile <= ws_floats, "step GEMM: partial workspace too small");
    FSB_CUDA(cudaMalloc(&plan->sched_dev, items.size() * sizeof(int4)));
    FSB_CUDA(cudaMemcpy(plan->sched_dev, items.data(), items.size() * sizeof(int4), cudaMemcpyHostToDevice));
    FSB_CUDA(cudaMalloc(&plan->cta_items_dev, cta_items.size() * sizeof(int)));
    FSB_CUDA(cudaMemcpy(plan->cta_items_dev, cta_items.data(), cta_items.size() * sizeof(int), cudaMemcpyHostToDevice));
    FSB_CUDA(cudaMalloc(&plan->nparts_dev, tiles * sizeof(int)));
    FSB_CUDA(cudaMemcpy(plan->nparts_dev, nparts.data(), tiles * sizeof(int), cudaMemcpyHostToDevice));
    StepGemmParams& p = plan->p;
    p.sched = reinterpret_cast<const int4*>(plan->sched_dev);
    p.cta_items = plan->cta_items_dev;
    p.tiles = tiles;
    p.stages = stages;
    p.n_out = n_out;
    p.K = K;
    p.a_hint = kEvictFirst;  // weights are streamed once per step (>> L2)
    p.b_hint = kEvictLast;   // the activation tile is re-read by every CTA
    p.ws = ws;
    plan->grid = dim3(static_cast<unsigned>(num_ctas), 1, 1);
    plan->smem = smem_of(stages);
    plan->norm = norm;
    plan->rt = row_tile;
    plan->weight_bytes = static_cast<double>(n_out) * K * 2;
    return 0;
}

StepPartials step_plan_partials(const StepGemmPlan& plan) {
    StepPartials P;
    P.ws = plan.p.ws;
    P.nparts = plan.nparts_dev;
    P.tiles = plan.p.tiles;
    P.n_out = plan.p.n_out;
    P.max_parts = plan.max_parts;
    P.rt = plan.rt;
    return P;
}

StepFinalize step_finalize_resid(const StepGemmPlan& src, const __nv_bfloat16* bias, const __nv_bfloat16* resid,
                                 __nv_bfloat16* x_out, float* ssq_out) {
    StepFinalize f{};
    f.pro = PRO_RESID;
    f.prev = step_plan_partials(src);
    f.bias = bias;
    f.resid = resid;
    f.x_out = x_out;
    f.ssq_out = ssq_out;
    return f;
}

StepFinalize step_finalize_swiglu(const StepGemmPlan& src, __nv_bfloat16* h, int I) {
    StepFinalize f{};
    f.pro = PRO_SWIGLU;
    f.prev = step_plan_partials(src);
    f.h = h;
    f.I = I;
    return f;
}

void step_plan_free(StepGemmPlan* plan) {
    if (plan->sched_dev) cudaFree(plan->sched_dev);
    if (plan->cta_items_dev) cudaFree(plan->cta_items_dev);
    if (plan->nparts_dev) cudaFree(plan->nparts_dev);
    plan->sched_dev = nullptr;
    plan->cta_items_dev = nullptr;
    plan->nparts_dev = nullptr;
}

namespace {
template <int PRO, int RT>
int finalize_t(const StepFinalize& p, cudaStream_t st) {
    const dim3 units(p.prev.tiles * cdiv(p.rows, kFinalizeRows<PRO>));
    FSB_LAUNCH((step_finalize_kernel<PRO, RT>), units, dim3(kEpiThreads), 0, st, p);
    return 0;
}
}  // namespace

int step_finalize_launch(const StepFinalize& fin, int rows, cudaStream_t st) {
    StepFinalize p = fin;
    p.rows = rows;
    if (p.prev.rt == kStepRowsMax)
        return p.pro == PRO_RESID ? finalize_t<PRO_RESID, kStepRowsMax>(p, st) : finalize_t<PRO_SWIGLU, kStepRowsMax>(p, st);
    return p.pro == PRO_RESID ? finalize_t<PRO_RESID, kStepRows>(p, st) : finalize_t<PRO_SWIGLU, kStepRows>(p, st);
}

int step_gemm_launch(const StepGemmPlan& plan, int rows, cudaStream_t st) {
    StepGemmParams p = plan.p;
    p.rows = rows;
    if (plan.rt == kStepRowsMax)
        return plan.norm ? launch_t<1, kStepRowsMax>(plan, p, st) : launch_t<0, kStepRowsMax>(plan, p, st);
    return plan.norm ? launch_t<1, kStepRows>(plan, p, st) : launch_t<0, kStepRows>(plan, p, st);
}

}  // namespace fsb
