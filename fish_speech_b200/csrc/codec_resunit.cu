// One decoder ResidualUnit of the codec as ONE kernel (modded_dac.py:599-620; dac ResidualUnit):
//
//     y = x + conv1( snake_1( conv7_dilated( snake_0(x) ) ) )
//
// Inputs are what the producing layer left behind: the raw residual stream x and its Snake-activated copy
// a = snake_0(x) (channels-last bf16 [B][T][C]).  Outputs: the new raw stream y (in place over x, optional) and
// snake_next(y) for the consumer, in a different buffer than `a` (neighbouring tiles still read their halo from `a`).
//
// Per tile of BM time steps (128; 64 for C = 384, whose accumulators take two warpgroups per 64 rows) -- one CTA per
// SM, persistent over the tiles:
//   phase 1  acc[128 x C]  = sum over 7 taps, C/64 k-blocks of  A(tap) W7(tap)^T : implicit im2col, the A tile of a
//            tap is fetched by TMA at a shifted time coordinate, rows before t = 0 are zero-filled by the TMA unit
//            (the causal left pad, modded_dac.py:546-552); wgmma, accumulator in registers.
//   epi 1    h = snake_1(acc + b7) -> bf16, written straight into shared memory in the K-major SWIZZLE_128B layout
//            the tensor core reads operand A in (fence.proxy.async): the intermediate never leaves the SM.
//   phase 2  acc[128 x C]  = h W1^T  (operand A from shared memory, W1 tiles through the same TMA ring).
//   epi 2    y = acc + b1 + x;  y and snake_next(y) are staged in shared memory (swizzled 64-channel blocks; the h buffer
//            is free again by then) and leave by TMA bulk tensor stores: whole 128-byte lines, issued asynchronously,
//            overlapping the next tile's first phase.  (C = 384: both staging buffers do not fit next to the ring;
//            that size stores from registers.)
// Against two separate GEMM launches this saves the write + read of h and of the 1x1 conv's operand
// (2 x 2 x N x C bytes of HBM traffic per unit) and one kernel's worth of residual-stream epilogue.
// Warpgroup g computes rows [64 (g % MH), +64) x channels [NB (g / MH), +NB) of both products (MH = BM / 64) and runs
// their epilogues;
// the last warp is the TMA producer, which runs ahead into the next tile while the epilogues run.
#include "gemm_tc.cuh"
#include "wgmma.cuh"

#include <cstring>
#include <map>
#include <mutex>

namespace fsb {

namespace {

constexpr int kRuTaps = 7;

struct ResUnitParams {
    int T, B;            // time steps per batch item, batch items
    int tiles_t, total;  // tiles per batch item, all tiles
    int stages;
    int shift[kRuTaps];  // time shift of tap q: -(6 - q) * dilation
    const float* b7;
    const float* alpha1;
    const float* inv1;
    const float* b1;
    const __nv_bfloat16* x;   // [B][T][C] raw residual stream
    __nv_bfloat16* out0;      // new raw stream (may alias x) or null
    __nv_bfloat16* out1;      // snake_next(y)
    const float* alpha_n;
    const float* inv_n;
};

__device__ __forceinline__ float ru_snake(float v, float a, float ia) {
    const float s = __sinf(a * v);
    return fmaf(ia * s, s, v);
}

template <int C>
struct RuShape {
    static constexpr int CP = (C + 63) / 64 * 64;   // K of both convolutions per tap, padded to the 64-wide k-block
    static constexpr int KB = CP / 64;
    static constexpr int NB = C <= 256 ? C : C / 2; // wgmma N (<= 256): wider outputs are split over warpgroups
    static constexpr int NS = C / NB;
    static constexpr int BM = NS == 1 ? 128 : 64;   // time steps per tile: the accumulators must fit the registers
    static constexpr int MH = BM / 64;
    static constexpr int kWarpgroups = MH * NS;     // 64-row blocks of the tile x channel blocks
    static constexpr int kABytes = BM * kBlockK * 2;
    static constexpr int kMmaThreads = kWarpgroups * 128;
    static constexpr int kThreads = kMmaThreads + 32;  // + the TMA producer warp
    static constexpr int kBBytes = C * kBlockK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kHBytes = KB * kABytes;
    static constexpr bool kStaged = C <= 192;  // outputs staged in shared memory and stored by TMA
    static constexpr int kY0Bytes = kStaged ? KB * kABytes : 0;
    static constexpr int kQ1 = 7 * KB;           // k-blocks of phase 1
    static_assert(C % 32 == 0 && NB % 16 == 0 && NB <= 256 && C <= 512, "channel count not supported");
};

__device__ __forceinline__ void ru_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// byte offset of (row r, channel c) in a [KB][BM rows][128 B] SWIZZLE_128B staging buffer (c even: a bf16 pair)
template <int BM>
__device__ __forceinline__ int ru_swz(int r, int c) {
    return (c >> 6) * (BM * 128) + r * 128 + (((((c & 63) >> 3) ^ (r & 7))) << 4) + (c & 7) * 2;
}

template <int C>
__global__ void __launch_bounds__(RuShape<C>::kThreads, 1)
res_unit_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW7,
                const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmY0,
                const __grid_constant__ CUtensorMap tmY1, const __grid_constant__ ResUnitParams p) {
    using S = RuShape<C>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t tiles = (raw + 1023u) & ~1023u;
    const int stages = p.stages;
    const uint32_t h_smem = tiles + static_cast<uint32_t>(stages) * S::kStageBytes;  // [KB][BM rows][128 B]
    const uint32_t y0_smem = h_smem + S::kHBytes;  // staging of the raw output (kStaged)
    const uint32_t bars = y0_smem + S::kY0Bytes;
    const uint32_t full0 = bars, empty0 = bars + 8u * stages;
    uint8_t* h_ptr = smem_raw + (h_smem - raw);
    uint8_t* y0_ptr = smem_raw + (y0_smem - raw);
    constexpr int kProducerWarp = S::kMmaThreads / 32;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int item_begin = static_cast<int>(static_cast<long long>(p.total) * blockIdx.x / gridDim.x);
    const int item_end = static_cast<int>(static_cast<long long>(p.total) * (blockIdx.x + 1) / gridDim.x);

    if (warp == kProducerWarp && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmW7);
        tma_prefetch_desc(&tmW1);
        for (int s = 0; s < stages; ++s) {
            mbar_init(full0 + 8u * s, 1);
            mbar_init(empty0 + 8u * s, kProducerWarp);  // one arrival per MMA warp
        }
        fence_mbar_init();
    }
    if (S::CP != C) {
        // channels C..CP-1 of h are K padding: zero once (W1's padding columns are zero as well, but 0 x NaN is NaN)
        for (int i = threadIdx.x; i < S::kHBytes / 16; i += S::kThreads) reinterpret_cast<uint4*>(h_ptr)[i] = make_uint4(0, 0, 0, 0);
        fence_proxy_async();
    }
    __syncthreads();

    pdl_launch_dependents();
    if (warp == kProducerWarp) {
        // ===== TMA producer: feeds the ring in exactly the order the MMA warpgroups consume it =====
        if (lane == 0) {
            pdl_wait();
            int it = 0;
            for (int n = item_begin; n < item_end; ++n) {
                const int z = n / p.tiles_t;
                const int t0 = (n - z * p.tiles_t) * S::BM;
                for (int q = 0; q < S::kQ1; ++q, ++it) {  // conv7: activations of the tap + its weights
                    const int s = it % stages;
                    const uint32_t dst = tiles + static_cast<uint32_t>(s) * S::kStageBytes;
                    mbar_wait(empty0 + 8u * s, (static_cast<uint32_t>(it / stages) & 1u) ^ 1u);
                    const int tap = q / S::KB, kb = q - tap * S::KB;
                    mbar_expect_tx(full0 + 8u * s, S::kStageBytes);
                    tma_load_3d(dst, &tmA, full0 + 8u * s, kb * kBlockK, t0 + p.shift[tap], z, kEvictNormal);
#pragma unroll
                    for (int hh = 0; hh < S::NS; ++hh)
                        tma_load_3d(dst + S::kABytes + hh * S::NB * 128, &tmW7, full0 + 8u * s,
                                    tap * S::CP + kb * kBlockK, hh * S::NB, 0, kEvictLast);
                }
                for (int kb = 0; kb < S::KB; ++kb, ++it) {  // conv1: its weights only (operand A is h in shared memory)
                    const int s = it % stages;
                    const uint32_t dst = tiles + static_cast<uint32_t>(s) * S::kStageBytes;
                    mbar_wait(empty0 + 8u * s, (static_cast<uint32_t>(it / stages) & 1u) ^ 1u);
                    mbar_expect_tx(full0 + 8u * s, S::kBBytes);
#pragma unroll
                    for (int hh = 0; hh < S::NS; ++hh)
                        tma_load_3d(dst + S::kABytes + hh * S::NB * 128, &tmW1, full0 + 8u * s, kb * kBlockK,
                                    hh * S::NB, 0, kEvictLast);
                }
            }
        }
    } else {
        // ===== MMA warpgroups =====
        const int wg = warp >> 2, wq = warp & 3;
        const int mh = wg % S::MH, cbase = (wg / S::MH) * S::NB;  // 64-row block of the tile, first channel
        const int r0 = mh * 64 + wq * 16 + (lane >> 2);     // tile rows r0 and r0 + 8 of this thread
        int it = 0;
        // k-blocks [0, nkb) of one product into d; operand A at a_of(q) (+ this warpgroup's 64-row half)
        auto run = [&](float* d, int nkb, auto a_of) {
#pragma unroll 1
            for (int q = 0; q < nkb; ++q, ++it) {
                const int s = it % stages;
                mbar_wait(full0 + 8u * s, static_cast<uint32_t>(it / stages) & 1u);
                const uint32_t src = tiles + static_cast<uint32_t>(s) * S::kStageBytes;
                const uint64_t ad = make_gdesc(a_of(q, src) + mh * kHalfATileBytes);
                const uint64_t bd = make_gdesc(src + S::kABytes + cbase * 128);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kBlockK / 16; ++k) wgmma_bf16<S::NB>(d, ad + 2u * k, bd + 2u * k, 1);
                wgmma_commit();
                wgmma_wait<1>();  // the previous k-block's MMAs have retired: release its ring slot
                if (q > 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(empty0 + 8u * ((it - 1) % stages));
                }
            }
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(empty0 + 8u * ((it - 1) % stages));
        };
        for (int n = item_begin; n < item_end; ++n) {
            const int z = n / p.tiles_t;
            const int t0 = (n - z * p.tiles_t) * S::BM;
            float d[S::NB / 2];
            // ---- phase 1: conv7 ----
#pragma unroll
            for (int e = 0; e < S::NB / 2; ++e) d[e] = 0.f;
            run(d, S::kQ1, [](int, uint32_t src) { return src; });
            // the previous tile's bulk stores read the h / y0 buffers: they must have finished reading
            if (S::kStaged && n > item_begin && threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            ru_bar(1, S::kMmaThreads);
            // ---- epilogue 1: h = snake_1(conv7 + b7) into the swizzled operand tile ----
#pragma unroll
            for (int b = 0; b < S::NB / 8; ++b) {
                const int c = cbase + 8 * b + 2 * (lane & 3);
                const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b7 + c));
                const float2 al = __ldg(reinterpret_cast<const float2*>(p.alpha1 + c));
                const float2 ia = __ldg(reinterpret_cast<const float2*>(p.inv1 + c));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = r0 + 8 * h;
                    // the unfused path stores conv7's output as bf16 only after the Snake: same rounding point here
                    *reinterpret_cast<uint32_t*>(h_ptr + ru_swz<S::BM>(r, c)) =
                        pack_bf2(ru_snake(d[4 * b + 2 * h] + bb.x, al.x, ia.x), ru_snake(d[4 * b + 2 * h + 1] + bb.y, al.y, ia.y));
                }
            }
            fence_proxy_async();  // generic-proxy writes of h -> visible to the tensor core's async proxy
            ru_bar(1, S::kMmaThreads);
            // ---- phase 2: conv1 over h ----
#pragma unroll
            for (int e = 0; e < S::NB / 2; ++e) d[e] = 0.f;
            run(d, S::KB, [&](int q, uint32_t) { return h_smem + static_cast<uint32_t>(q) * S::kABytes; });
            ru_bar(1, S::kMmaThreads);  // every warpgroup is done reading h before it takes snake_next(y)
            // ---- epilogue 2: y = conv1 + b1 + x; store y and snake_next(y) ----
#pragma unroll
            for (int b = 0; b < S::NB / 8; ++b) {
                const int c = cbase + 8 * b + 2 * (lane & 3);
                const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b1 + c));
                const float2 al = __ldg(reinterpret_cast<const float2*>(p.alpha_n + c));
                const float2 ia = __ldg(reinterpret_cast<const float2*>(p.inv_n + c));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = r0 + 8 * h;
                    const int t = t0 + r;
                    const bool live = t < p.T;
                    const size_t off = (static_cast<size_t>(z) * p.T + t) * C + c;
                    const uint32_t xr = live ? *reinterpret_cast<const uint32_t*>(p.x + off) : 0u;
                    // (acc + bias) + x, the association of the two-launch path: identical bits
                    const float f0 = (d[4 * b + 2 * h] + bb.x) + bf_lo(xr);
                    const float f1 = (d[4 * b + 2 * h + 1] + bb.y) + bf_hi(xr);
                    const uint32_t y = pack_bf2(f0, f1);
                    const uint32_t ys = pack_bf2(ru_snake(f0, al.x, ia.x), ru_snake(f1, al.y, ia.y));
                    if (S::kStaged) {
                        if (p.out0) *reinterpret_cast<uint32_t*>(y0_ptr + ru_swz<S::BM>(r, c)) = y;
                        *reinterpret_cast<uint32_t*>(h_ptr + ru_swz<S::BM>(r, c)) = ys;  // h has been consumed by phase 2
                    } else if (live) {
                        if (p.out0) *reinterpret_cast<uint32_t*>(p.out0 + off) = y;
                        *reinterpret_cast<uint32_t*>(p.out1 + off) = ys;
                    }
                }
            }
            if (S::kStaged) {
                fence_proxy_async();  // the staged tiles -> visible to the TMA engine
                ru_bar(1, S::kMmaThreads);
                if (threadIdx.x == 0) {
#pragma unroll
                    for (int kb = 0; kb < S::KB; ++kb) {
                        if (p.out0) tma_store_3d(&tmY0, y0_smem + kb * S::kABytes, kb * kBlockK, t0, z);
                        tma_store_3d(&tmY1, h_smem + kb * S::kABytes, kb * kBlockK, t0, z);
                    }
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if (S::kStaged && threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores complete
    }
}

struct RuKey {
    const void *a, *w7, *w1, *out0, *out1;
    int B, T, C, dil;
    bool operator<(const RuKey& o) const {
        return memcmp(this, &o, sizeof(RuKey)) < 0;
    }
};
struct RuPlan {
    CUtensorMap tmA, tmW7, tmW1, tmY0, tmY1;
    int stages;
    size_t smem;
    dim3 grid;
};
std::mutex g_ru_mutex;
std::map<RuKey, RuPlan> g_ru_plans;
constexpr size_t kMaxRuPlans = 256;

template <int C>
int ru_setup() {
    static bool done = false;
    if (done) return 0;
    FSB_CUDA(cudaFuncSetAttribute(res_unit_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    FSB_CUDA(cudaFuncSetAttribute(res_unit_kernel<C>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                  cudaSharedmemCarveoutMaxShared));
    done = true;
    return 0;
}

template <int C>
int ru_launch(const RuPlan& plan, const ResUnitParams& p, cudaStream_t st) {
    FSB_TRY(ru_setup<C>());
    FSB_LAUNCH(res_unit_kernel<C>, plan.grid, dim3(RuShape<C>::kThreads), plan.smem, st, plan.tmA, plan.tmW7, plan.tmW1, plan.tmY0,
               plan.tmY1, p);
    return 0;
}

template <int C>
int ru_plan(RuPlan* plan, const void* a, const void* w7, const void* w1, const void* out0, const void* out1, int B, int T) {
    using S = RuShape<C>;
    GemmOperand A{reinterpret_cast<const __nv_bfloat16*>(a), C, T, B, C, static_cast<long long>(T) * C};
    GemmOperand W7{reinterpret_cast<const __nv_bfloat16*>(w7), static_cast<long long>(kRuTaps) * S::CP, C, 1,
                   static_cast<long long>(kRuTaps) * S::CP, static_cast<long long>(C) * kRuTaps * S::CP};
    GemmOperand W1{reinterpret_cast<const __nv_bfloat16*>(w1), S::CP, C, 1, S::CP, static_cast<long long>(C) * S::CP};
    FSB_TRY(gemm_make_tmap(&plan->tmA, A, S::BM));
    FSB_TRY(gemm_make_tmap(&plan->tmW7, W7, S::NB));
    FSB_TRY(gemm_make_tmap(&plan->tmW1, W1, S::NB));
    // outputs: the same {64 channels, BM time steps} boxes, written by TMA from the staging tiles
    GemmOperand Y1 = A, Y0 = A;
    Y1.ptr = reinterpret_cast<const __nv_bfloat16*>(out1);
    Y0.ptr = reinterpret_cast<const __nv_bfloat16*>(out0 ? out0 : out1);
    FSB_TRY(gemm_make_tmap(&plan->tmY1, Y1, S::BM));
    FSB_TRY(gemm_make_tmap(&plan->tmY0, Y0, S::BM));
    const int budget = 227 * 1024 - 1024 - 256 - S::kHBytes - S::kY0Bytes;
    int stages = budget / S::kStageBytes;
    if (stages > 6) stages = 6;
    FSB_CHECK(stages >= 2, "res_unit: not enough shared memory for C=%d", C);
    plan->stages = stages;
    plan->smem = static_cast<size_t>(stages) * S::kStageBytes + S::kHBytes + S::kY0Bytes + 1024 + 16 * stages + 64;
    int dev = 0, sms = 0;
    FSB_CUDA(cudaGetDevice(&dev));
    FSB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const long long total = static_cast<long long>(B) * cdiv(T, S::BM);
    plan->grid = dim3(static_cast<unsigned>(total < sms ? total : sms), 1, 1);
    return 0;
}

}  // namespace

bool res_unit_supported(int C) { return C == 96 || C == 192 || C == 384; }

int res_unit_run(const void* d_a, const void* d_x, int B, int T, int C, int dilation, const void* d_w7,
                 const float* d_b7, const float* d_alpha1, const float* d_inv1, const void* d_w1, const float* d_b1,
                 void* d_out0, void* d_out1, const float* d_alpha_n, const float* d_inv_n, cudaStream_t st) {
    FSB_CHECK(res_unit_supported(C), "res_unit: C=%d not supported", C);
    FSB_CHECK(d_out1 != nullptr && d_out1 != d_a, "res_unit: the activated output must not alias the activated input");
    FSB_CHECK(d_b7 && d_b1 && d_alpha1 && d_inv1 && d_alpha_n && d_inv_n, "res_unit: missing per-channel vector");
    RuKey key;
    memset(&key, 0, sizeof(key));
    key.a = d_a; key.w7 = d_w7; key.w1 = d_w1; key.out0 = d_out0; key.out1 = d_out1;
    key.B = B; key.T = T; key.C = C; key.dil = dilation;
    RuPlan plan;
    {
        std::lock_guard<std::mutex> lk(g_ru_mutex);
        auto it = g_ru_plans.find(key);
        if (it == g_ru_plans.end()) {
            RuPlan np;
            memset(&np, 0, sizeof(np));
            int rc = C == 96 ? ru_plan<96>(&np, d_a, d_w7, d_w1, d_out0, d_out1, B, T)
                             : (C == 192 ? ru_plan<192>(&np, d_a, d_w7, d_w1, d_out0, d_out1, B, T)
                                         : ru_plan<384>(&np, d_a, d_w7, d_w1, d_out0, d_out1, B, T));
            if (rc) return rc;
            if (g_ru_plans.size() >= kMaxRuPlans) g_ru_plans.clear();
            it = g_ru_plans.emplace(key, np).first;
        }
        plan = it->second;
    }
    ResUnitParams p;
    memset(&p, 0, sizeof(p));
    p.T = T; p.B = B;
    p.tiles_t = cdiv(T, C == 384 ? RuShape<384>::BM : kBlockM);
    p.total = B * p.tiles_t;
    p.stages = plan.stages;
    for (int q = 0; q < kRuTaps; ++q) p.shift[q] = -(kRuTaps - 1 - q) * dilation;
    p.b7 = d_b7; p.alpha1 = d_alpha1; p.inv1 = d_inv1; p.b1 = d_b1;
    p.x = reinterpret_cast<const __nv_bfloat16*>(d_x);
    p.out0 = reinterpret_cast<__nv_bfloat16*>(d_out0);
    p.out1 = reinterpret_cast<__nv_bfloat16*>(d_out1);
    p.alpha_n = d_alpha_n; p.inv_n = d_inv_n;
    switch (C) {
        case 96: return ru_launch<96>(plan, p, st);
        case 192: return ru_launch<192>(plan, p, st);
        default: return ru_launch<384>(plan, p, st);
    }
}

}  // namespace fsb
