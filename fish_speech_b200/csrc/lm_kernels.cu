// See lm_kernels.cuh.  All kernels here are HBM/L2-bound glue: vectorised, coalesced, warp-shuffle
// reductions, fp32 math with bf16 rounding at the reference's rounding points.
#include "lm_kernels.cuh"

namespace fsb {

namespace {

// Sum of squares of 4 consecutive features per lane over one 128-feature tile -> all lanes.
__device__ __forceinline__ float tile_ssq(const float (&x)[4]) {
    return warp_sum(((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]) + x[3] * x[3]);
}

// ------------------------------------------------------------------------------------------------
// embed: llama.py:399-420 (+ per-tile sum of squares for the first layer's normalise-on-load)
// ------------------------------------------------------------------------------------------------
constexpr int kRowThreads = 256;

__global__ void __launch_bounds__(kRowThreads) embed_kernel(EmbedArgs a, float inv_div) {
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int* t = a.tokens + static_cast<size_t>(row) * (a.C + 1);
    int tok = t[0];
    const bool sem = tok >= a.sem_begin && tok <= a.sem_end;
    tok = min(max(tok, 0), a.vocab - 1);
    const int nt = (a.D + kSsqTile - 1) / kSsqTile;
    for (int tile = warp; tile < nt; tile += kRowThreads / 32) {
        const int f = tile * kSsqTile + lane * 4;
        float x[4] = {0.f, 0.f, 0.f, 0.f};
        if (f < a.D) {  // D % 4 == 0
            float s[4] = {0.f, 0.f, 0.f, 0.f};
            if (sem) {
                for (int c = 0; c < a.C; ++c) {
                    const int code = min(max(t[c + 1], 0), a.cs - 1);
                    const uint2 u = *reinterpret_cast<const uint2*>(a.cb_emb + (static_cast<size_t>(c) * a.cs + code) * a.D + f);
                    s[0] += bf_lo(u.x); s[1] += bf_hi(u.x); s[2] += bf_lo(u.y); s[3] += bf_hi(u.y);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) s[q] = rbf(s[q]);  // torch.stack(...).sum(dim=1) -> one bf16 rounding
            }
            const uint2 e = *reinterpret_cast<const uint2*>(a.emb + static_cast<size_t>(tok) * a.D + f);
            const float ev[4] = {bf_lo(e.x), bf_hi(e.x), bf_lo(e.y), bf_hi(e.y)};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                x[q] = rbf(ev[q] + s[q]);
                if (sem && a.scale) x[q] = rbf(x[q] / inv_div);  // x / sqrt(C+1)
            }
            uint2 o;
            o.x = pack_bf2(x[0], x[1]);
            o.y = pack_bf2(x[2], x[3]);
            *reinterpret_cast<uint2*>(a.x + static_cast<size_t>(row) * a.D + f) = o;
        }
        const float ss = tile_ssq(x);
        if (a.ssq != nullptr && lane == 0) a.ssq[row * kSsqRowStride + tile] = ss;
    }
}

// ------------------------------------------------------------------------------------------------
// rows: gather (+ fish RMSNorm) of whole rows into a residual stream, with its per-tile sum of squares
// ------------------------------------------------------------------------------------------------
constexpr int kRowsMaxTilesPerWarp = 4;  // D <= 4096 with 8 warps

__global__ void __launch_bounds__(kRowThreads) rows_kernel(RowsArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m = a.gather_map ? a.gather_map[row] : row;
    const int src = a.gather ? a.gather[static_cast<size_t>(m) * a.gather_stride] : row;
    const int nt = (a.D + kSsqTile - 1) / kSsqTile;
    float x[kRowsMaxTilesPerWarp][4];
#pragma unroll
    for (int e = 0; e < kRowsMaxTilesPerWarp; ++e) {
        const int tile = warp + e * (kRowThreads / 32);
        const int f = tile * kSsqTile + lane * 4;
        x[e][0] = x[e][1] = x[e][2] = x[e][3] = 0.f;
        if (tile < nt && f < a.D) {
            const uint2 u = *reinterpret_cast<const uint2*>(a.x + static_cast<size_t>(src) * a.D + f);
            x[e][0] = bf_lo(u.x); x[e][1] = bf_hi(u.x); x[e][2] = bf_lo(u.y); x[e][3] = bf_hi(u.y);
        }
    }
    float r = 1.f;
    if (a.norm_w != nullptr) {
        // the row's sum of squares as the producing kernel left it, added tile by tile in tile order: exactly
        // what the step GEMM's normalise-on-load computes, so both see the same rsqrt
        const float* q = a.ssq_in + static_cast<size_t>(src) * kSsqRowStride;
        float tot = 0.f;
        for (int t = 0; t < nt; ++t) tot += q[t];
        r = rsqrtf(tot / static_cast<float>(a.D) + a.eps);
    }
#pragma unroll
    for (int e = 0; e < kRowsMaxTilesPerWarp; ++e) {
        const int tile = warp + e * (kRowThreads / 32);
        const int f = tile * kSsqTile + lane * 4;
        const bool live = tile < nt && f < a.D;
        if (live && a.norm_w != nullptr) {
            const uint2 w = *reinterpret_cast<const uint2*>(a.norm_w + f);
            const float wf[4] = {bf_lo(w.x), bf_hi(w.x), bf_lo(w.y), bf_hi(w.y)};
#pragma unroll
            for (int q = 0; q < 4; ++q) x[e][q] = rbf(rbf(x[e][q] * r) * wf[q]);
        }
        if (live) {
            uint2 o;
            o.x = pack_bf2(x[e][0], x[e][1]);
            o.y = pack_bf2(x[e][2], x[e][3]);
            *reinterpret_cast<uint2*>(a.y + static_cast<size_t>(row) * a.D + f) = o;
        }
        if (tile < nt) {
            const float ss = tile_ssq(x[e]);
            if (a.ssq != nullptr && lane == 0) a.ssq[row * kSsqRowStride + tile] = ss;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// residual add + fish RMSNorm on a plain fp32 GEMM result (prefill, codec transformer)
// ------------------------------------------------------------------------------------------------
constexpr int kRnThreads = 512;
constexpr int kRnMaxPer = 8;  // D <= 4096

__global__ void __launch_bounds__(kRnThreads) resid_norm_kernel(ResidNormArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float red[33];
    const int row = blockIdx.x;
    float v[kRnMaxPer];
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < kRnMaxPer; ++e) {
        const int f = threadIdx.x + e * kRnThreads;
        v[e] = 0.f;
        if (f < a.D) {
            float x = a.x_in ? bf2f(a.x_in[static_cast<size_t>(row) * a.D + f]) : 0.f;
            if (a.y) {
                float yy = a.y[static_cast<size_t>(row) * a.ld + f];
                if (a.bias) yy += bf2f(a.bias[f]);
                yy = rbf(yy);
                if (a.scale) yy *= bf2f(a.scale[f]);
                x = rbf(x + yy);
            }
            v[e] = x;
            ss += x * x;
            if (a.x_out) a.x_out[static_cast<size_t>(row) * a.D + f] = f2bf(x);
        }
    }
    if (a.norm_w != nullptr) {
        const float tot = block_sum(ss, red);
        const float r = rsqrtf(tot / static_cast<float>(a.D) + a.eps);
#pragma unroll
        for (int e = 0; e < kRnMaxPer; ++e) {
            const int f = threadIdx.x + e * kRnThreads;
            if (f < a.D) a.n_out[static_cast<size_t>(row) * a.D + f] = f2bf(rbf(rbf(v[e] * r) * bf2f(a.norm_w[f])));
        }
    }
}

// Vectorised form (D % 4 == 0, ld % 4 == 0): 4 consecutive features per thread, 16-byte loads of y.
constexpr int kRn4Threads = 256;
constexpr int kRn4MaxPer = 4;  // D <= 4096
__global__ void __launch_bounds__(kRn4Threads) resid_norm4_kernel(ResidNormArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float red[33];
    const int row = blockIdx.x;
    float v[kRn4MaxPer][4];
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < kRn4MaxPer; ++e) {
        const int f = (threadIdx.x + e * kRn4Threads) * 4;
        v[e][0] = v[e][1] = v[e][2] = v[e][3] = 0.f;
        if (f >= a.D) continue;
        float x[4] = {0.f, 0.f, 0.f, 0.f};
        if (a.x_in) {
            const uint2 u = *reinterpret_cast<const uint2*>(a.x_in + static_cast<size_t>(row) * a.D + f);
            x[0] = bf_lo(u.x); x[1] = bf_hi(u.x); x[2] = bf_lo(u.y); x[3] = bf_hi(u.y);
        }
        if (a.y) {
            const float4 y4 = *reinterpret_cast<const float4*>(a.y + static_cast<size_t>(row) * a.ld + f);
            float yy[4] = {y4.x, y4.y, y4.z, y4.w};
            if (a.bias) {
                const uint2 b = *reinterpret_cast<const uint2*>(a.bias + f);
                yy[0] += bf_lo(b.x); yy[1] += bf_hi(b.x); yy[2] += bf_lo(b.y); yy[3] += bf_hi(b.y);
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) yy[c] = rbf(yy[c]);
            if (a.scale) {
                const uint2 sc = *reinterpret_cast<const uint2*>(a.scale + f);
                yy[0] *= bf_lo(sc.x); yy[1] *= bf_hi(sc.x); yy[2] *= bf_lo(sc.y); yy[3] *= bf_hi(sc.y);
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) x[c] = rbf(x[c] + yy[c]);
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            v[e][c] = x[c];
            ss += x[c] * x[c];
        }
        if (a.x_out) {
            uint2 o;
            o.x = pack_bf2(x[0], x[1]);
            o.y = pack_bf2(x[2], x[3]);
            *reinterpret_cast<uint2*>(a.x_out + static_cast<size_t>(row) * a.D + f) = o;
        }
    }
    if (a.norm_w != nullptr) {
        const float tot = block_sum(ss, red);
        const float r = rsqrtf(tot / static_cast<float>(a.D) + a.eps);
#pragma unroll
        for (int e = 0; e < kRn4MaxPer; ++e) {
            const int f = (threadIdx.x + e * kRn4Threads) * 4;
            if (f >= a.D) continue;
            const uint2 w = *reinterpret_cast<const uint2*>(a.norm_w + f);
            const float wf[4] = {bf_lo(w.x), bf_hi(w.x), bf_lo(w.y), bf_hi(w.y)};
            float n[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) n[c] = rbf(rbf(v[e][c] * r) * wf[c]);
            uint2 o;
            o.x = pack_bf2(n[0], n[1]);
            o.y = pack_bf2(n[2], n[3]);
            *reinterpret_cast<uint2*>(a.n_out + static_cast<size_t>(row) * a.D + f) = o;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// q/k/v post-processing: llama.py:891-911
// ------------------------------------------------------------------------------------------------
__global__ void qkv_prep_kernel(QkvPrepArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float red[33];
    const int row = blockIdx.x, head = blockIdx.y;
    const int t = threadIdx.x;  // pair index, Dh/2 threads
    const int Dh = a.Dh;
    const int kind = head < a.H ? 0 : (head < a.H + a.Hkv ? 1 : 2);  // q, k, v
    const int f0 = head * Dh + 2 * t;
    const float2 y2 = *reinterpret_cast<const float2*>(a.y + static_cast<size_t>(row) * a.ld + f0);
    float v0 = y2.x, v1 = y2.y;
    if (a.bias) {
        v0 += bf2f(a.bias[f0]);
        v1 += bf2f(a.bias[f0 + 1]);
    }
    v0 = rbf(v0);
    v1 = rbf(v1);
    const __nv_bfloat16* nw = kind == 0 ? a.q_norm : (kind == 1 ? a.k_norm : nullptr);
    if (nw != nullptr) {
        // nn.RMSNorm(head_dim): fp32 math, weight multiply included, ONE rounding
        const float tot = block_sum(v0 * v0 + v1 * v1, red);
        const float r = rsqrtf(tot / static_cast<float>(Dh) + a.eps);
        v0 = rbf(v0 * r * bf2f(nw[2 * t]));
        v1 = rbf(v1 * r * bf2f(nw[2 * t + 1]));
    }
    const int pos = a.row_pos[row];
    if (kind != 2) {
        const __nv_bfloat16* f = a.freqs + (static_cast<size_t>(max(pos, 0)) * (Dh / 2) + t) * 2;
        const float c = bf2f(f[0]), s = bf2f(f[1]);
        const float o0 = __fsub_rn(__fmul_rn(v0, c), __fmul_rn(v1, s));
        const float o1 = __fadd_rn(__fmul_rn(v1, c), __fmul_rn(v0, s));
        v0 = rbf(o0);
        v1 = rbf(o1);
    }
    const uint32_t packed = pack_bf2(v0, v1);
    if (kind == 0) {
        uint32_t* dst = reinterpret_cast<uint32_t*>(a.q + (static_cast<size_t>(row) * a.H + head) * Dh);
        dst[t] = packed;
    } else if (pos >= 0 && pos < a.S) {
        const int g = kind == 1 ? head - a.H : head - a.H - a.Hkv;
        __nv_bfloat16* cache = kind == 1 ? a.kcache : a.vcache;
        const long long off = kv_offset(a.kv_page, a.kv_page_ld, a.row_seq[row], g, pos, a.Hkv, a.S, Dh);
        if (off >= 0) reinterpret_cast<uint32_t*>(cache + off)[t] = packed;
    }
}

// The same per (row, head) work with one CTA per row: a warp takes whole heads (lane = rotary pair, two pairs per lane
// at head_dim 128), so the per-head norm is a warp reduction and a row costs one CTA of 8 warps instead of H + 2 Hkv
// CTAs of Dh / 2 threads (393 216 one-warp CTAs per codec transformer layer at 32 x 256 frames).
constexpr int kQkvRowThreads = 256;
template <int DH, bool RING>
__global__ void __launch_bounds__(kQkvRowThreads) qkv_prep_row_kernel(QkvPrepArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    constexpr int PPL = DH / 64;  // rotary pairs per lane
    const int row = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pos = a.row_pos[row];
    const int b = a.row_seq[row];
    const int NH = a.H + 2 * a.Hkv;
    for (int head = warp; head < NH; head += kQkvRowThreads / 32) {
        const int kind = head < a.H ? 0 : (head < a.H + a.Hkv ? 1 : 2);  // q, k, v
        const __nv_bfloat16* nw = kind == 0 ? a.q_norm : (kind == 1 ? a.k_norm : nullptr);
        float v0[PPL], v1[PPL];
        float ss = 0.f;
#pragma unroll
        for (int u = 0; u < PPL; ++u) {
            const int t = lane + 32 * u;
            const int f0 = head * DH + 2 * t;
            const float2 y2 = *reinterpret_cast<const float2*>(a.y + static_cast<size_t>(row) * a.ld + f0);
            v0[u] = y2.x;
            v1[u] = y2.y;
            if (a.bias) {
                v0[u] += bf2f(a.bias[f0]);
                v1[u] += bf2f(a.bias[f0 + 1]);
            }
            v0[u] = rbf(v0[u]);
            v1[u] = rbf(v1[u]);
            ss += v0[u] * v0[u] + v1[u] * v1[u];
        }
        if (nw != nullptr) {
            // nn.RMSNorm(head_dim): fp32 math, weight multiply included, ONE rounding
            const float r = rsqrtf(warp_sum(ss) / static_cast<float>(DH) + a.eps);
#pragma unroll
            for (int u = 0; u < PPL; ++u) {
                const int t = lane + 32 * u;
                v0[u] = rbf(v0[u] * r * bf2f(nw[2 * t]));
                v1[u] = rbf(v1[u] * r * bf2f(nw[2 * t + 1]));
            }
        }
#pragma unroll
        for (int u = 0; u < PPL; ++u) {
            const int t = lane + 32 * u;
            if (kind != 2) {
                const uint32_t cs = *reinterpret_cast<const uint32_t*>(a.freqs + (static_cast<size_t>(max(pos, 0)) * (DH / 2) + t) * 2);
                const float c = bf_lo(cs), sn = bf_hi(cs);
                const float o0 = __fsub_rn(__fmul_rn(v0[u], c), __fmul_rn(v1[u], sn));
                const float o1 = __fadd_rn(__fmul_rn(v1[u], c), __fmul_rn(v0[u], sn));
                v0[u] = rbf(o0);
                v1[u] = rbf(o1);
            }
            const uint32_t packed = pack_bf2(v0[u], v1[u]);
            if (kind == 0) {
                reinterpret_cast<uint32_t*>(a.q + (static_cast<size_t>(row) * a.H + head) * DH)[t] = packed;
            } else if (RING) {
                if (pos >= 0) {
                    const int g = kind == 1 ? head - a.H : head - a.H - a.Hkv;
                    __nv_bfloat16* cache = kind == 1 ? a.kcache : a.vcache;
                    const int r = pos % a.S;
                    const long long base = kv_ring_row(b, g, a.Hkv, a.S);
                    reinterpret_cast<uint32_t*>(cache + (base + r) * DH)[t] = packed;
                    if (r < kKvPage) reinterpret_cast<uint32_t*>(cache + (base + a.S + r) * DH)[t] = packed;  // mirror
                }
            } else if (pos >= 0 && pos < a.S) {
                const int g = kind == 1 ? head - a.H : head - a.H - a.Hkv;
                __nv_bfloat16* cache = kind == 1 ? a.kcache : a.vcache;
                const long long off = kv_offset(a.kv_page, a.kv_page_ld, b, g, pos, a.Hkv, a.S, DH);
                if (off >= 0) reinterpret_cast<uint32_t*>(cache + off)[t] = packed;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// length-aware GQA attention over the KV cache (one query token per CTA, all G heads of a KV group)
// ------------------------------------------------------------------------------------------------
constexpr int kAttnThreads = 256;
constexpr int kAttnWarps = kAttnThreads / 32;
constexpr int kAttnPrefetchPos = 2048;  // positions of K/V history the decode attention prefetches to L2 (8 lines per thread)

// Softmax(q k^T) v of one query token against positions [0, L) of one KV group: all G query heads of the group at once.
// The score buffer holds `lcap` positions per head (a multiple of 32).  A context that fits is scored once; a longer
// one is walked in chunks of lcap three times -- maximum, sum of exponentials, weighted values -- recomputing the
// scores each time.  Chunk boundaries are multiples of 32, so every lane and every warp accumulates exactly the
// sequence of terms it would in one pass: the result is bit-identical to the unchunked kernel, whatever lcap is.
// Row p of the history: kc + pt[p / kKvPage] * page_stride + (p % kKvPage) * DH, with `pt` the row's page-table entries
// in shared memory. A paged cache: kc / vc at this KV head's offset inside a page, page_stride elements between pages
// (kv_offset). A contiguous one: pt[j] = j and page_stride = kKvPage * DH, one code path for both.
template <int DH, int G>
__device__ __forceinline__ void attend(const float* qs, float* sc, float* red, const __nv_bfloat16* kc,
                                       const __nv_bfloat16* vc, const int* pt, size_t page_stride, int L, int lcap,
                                       float scale, int bf16_math, __nv_bfloat16* out) {
    static_assert(G <= kAttnWarps, "one warp per query head in the softmax");
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int LPR = DH / 8;    // lanes per cache row (16-byte loads)
    constexpr int RPW = 32 / LPR;  // rows per warp iteration
    constexpr int UNR = 4;         // independent 16-byte loads in flight per lane
    constexpr int DPL = DH / 32;   // value dims per lane
    const int sub = lane / LPR, li = lane % LPR;
    float qr[G][8];
#pragma unroll
    for (int gg = 0; gg < G; ++gg)
#pragma unroll
        for (int e = 0; e < 8; ++e) qr[gg][e] = qs[gg * DH + li * 8 + e];

    auto at = [&](const __nv_bfloat16* base, int p) {
        return base + static_cast<size_t>(pt[p / kKvPage]) * page_stride + (p % kKvPage) * DH;
    };
    auto scores = [&](int c0, int n) {  // sc[gg][p - c0] for p in [c0, c0 + n)
        for (int pb = warp * RPW * UNR; pb < n; pb += kAttnWarps * RPW * UNR) {
            uint4 u[UNR];
            const __nv_bfloat16* kp = at(kc, c0 + pb);  // RPW * UNR positions from a multiple of 8: one page
#pragma unroll
            for (int j = 0; j < UNR; ++j) {
                const int p = pb + j * RPW + sub;
                u[j] = make_uint4(0, 0, 0, 0);
                if (p < n) u[j] = *reinterpret_cast<const uint4*>(kp + (j * RPW + sub) * DH + li * 8);
            }
#pragma unroll
            for (int j = 0; j < UNR; ++j) {
                const int p = pb + j * RPW + sub;
                const bool ok = p < n;
                const float kf[8] = {bf_lo(u[j].x), bf_hi(u[j].x), bf_lo(u[j].y), bf_hi(u[j].y),
                                     bf_lo(u[j].z), bf_hi(u[j].z), bf_lo(u[j].w), bf_hi(u[j].w)};
#pragma unroll
                for (int gg = 0; gg < G; ++gg) {
                    float d = 0.f;
#pragma unroll
                    for (int e = 0; e < 8; ++e) d += qr[gg][e] * kf[e];
#pragma unroll
                    for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
                    if (ok && li == 0) sc[gg * lcap + p] = bf16_math ? rbf(rbf(d) * scale) : d * scale;
                }
            }
        }
        __syncthreads();
    };

    const bool one = L <= lcap;
    float m = -INFINITY, z = 0.f;  // of head `warp` (warps < G)
    if (one) {
        scores(0, L);
        if (warp < G) {
            float* s = sc + warp * lcap;
            for (int p = lane; p < L; p += 32) m = fmaxf(m, s[p]);
            m = warp_max(m);
            for (int p = lane; p < L; p += 32) {
                const float e = expf(s[p] - m);
                s[p] = e;
                z += e;
            }
            z = warp_sum(z);
            for (int p = lane; p < L; p += 32) {
                const float pr = s[p] / z;
                s[p] = bf16_math ? rbf(pr) : pr;
            }
        }
        __syncthreads();
    } else {
        for (int c0 = 0; c0 < L; c0 += lcap) {
            const int n = min(lcap, L - c0);
            scores(c0, n);
            if (warp < G)
                for (int p = lane; p < n; p += 32) m = fmaxf(m, sc[warp * lcap + p]);
            __syncthreads();
        }
        m = warp_max(m);
        for (int c0 = 0; c0 < L; c0 += lcap) {
            const int n = min(lcap, L - c0);
            scores(c0, n);
            if (warp < G)
                for (int p = lane; p < n; p += 32) z += expf(sc[warp * lcap + p] - m);
            __syncthreads();
        }
        z = warp_sum(z);
    }

    float acc[G][DPL];
#pragma unroll
    for (int gg = 0; gg < G; ++gg)
#pragma unroll
        for (int e = 0; e < DPL; ++e) acc[gg][e] = 0.f;
    for (int c0 = 0; c0 < L; c0 += lcap) {
        const int n = min(lcap, L - c0);
        if (!one) {
            scores(c0, n);
            if (warp < G) {
                float* s = sc + warp * lcap;
                for (int p = lane; p < n; p += 32) {
                    const float pr = expf(s[p] - m) / z;
                    s[p] = bf16_math ? rbf(pr) : pr;
                }
            }
            __syncthreads();
        }
        for (int pb = warp; pb < n; pb += kAttnWarps * UNR) {
            const __nv_bfloat16* vp = at(vc, c0 + pb);  // positions pb + 8 j, inside a run of 32 from a multiple of 32: one page
            float vf[UNR][DPL];
#pragma unroll
            for (int j = 0; j < UNR; ++j) {
                const int p = pb + j * kAttnWarps;
#pragma unroll
                for (int e = 0; e < DPL; ++e) vf[j][e] = 0.f;
                if (p < n) {
                    if (DPL == 4) {
                        const uint2 u2 = *reinterpret_cast<const uint2*>(vp + (j * kAttnWarps) * DH + lane * 4);
                        vf[j][0] = bf_lo(u2.x); vf[j][1] = bf_hi(u2.x); vf[j][2 % DPL] = bf_lo(u2.y); vf[j][3 % DPL] = bf_hi(u2.y);
                    } else {
                        const uint32_t u1 = *reinterpret_cast<const uint32_t*>(vp + (j * kAttnWarps) * DH + lane * 2);
                        vf[j][0] = bf_lo(u1); vf[j][1] = bf_hi(u1);
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < UNR; ++j) {
                const int p = pb + j * kAttnWarps;
                if (p < n) {
#pragma unroll
                    for (int gg = 0; gg < G; ++gg) {
                        const float w = sc[gg * lcap + p];
#pragma unroll
                        for (int e = 0; e < DPL; ++e) acc[gg][e] += w * vf[j][e];
                    }
                }
            }
        }
        if (!one) __syncthreads();  // the next chunk overwrites the scores
    }
#pragma unroll
    for (int gg = 0; gg < G; ++gg)
#pragma unroll
        for (int e = 0; e < DPL; ++e) red[(warp * G + gg) * DH + lane * DPL + e] = acc[gg][e];
    __syncthreads();
    for (int e = threadIdx.x; e < G * DH; e += kAttnThreads) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < kAttnWarps; ++w) s += red[w * G * DH + e];
        out[e] = f2bf(s);
    }
}


// RING: the cache is a ring (kv_ring_row); the "pages" are then the runs of kKvPage positions from lo, each one run of
// consecutive rows thanks to the mirror, so attend() walks the same positions in the same order as over a linear cache.
template <int DH, int G, bool RING>
__global__ void __launch_bounds__(kAttnThreads) attn_kernel(AttnArgs a, float scale, int lcap) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float sm[];
    float* qs = sm;                      // [G][DH]
    float* sc = qs + G * DH;             // [G][lcap]
    float* red = sc + G * lcap;          // [kAttnWarps][G][DH]
    const int row = blockIdx.y, g = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // a position past a linear cache reads its last row
    const int b = a.row_seq[row], pos = RING ? a.row_pos[row] : min(a.row_pos[row], a.S - 1);
    if (pos < 0) {  // idle slot parked at position -1: nothing to attend to
        for (int e = threadIdx.x; e < G * DH; e += kAttnThreads)
            a.out[(static_cast<size_t>(row) * a.H + blockIdx.x * G) * DH + e] = f2bf(0.f);
        return;
    }
    const int lo = (a.window > 0 && pos - a.window + 1 > 0) ? pos - a.window + 1 : 0;  // 0 when paged
    const int L = pos - lo + 1;
    int* pt = reinterpret_cast<int*>(red + kAttnWarps * G * DH);  // [pages of positions lo..pos]
    bool unmapped = false;
    for (int j = threadIdx.x; j <= (L - 1) / kKvPage; j += kAttnThreads) {
        if (RING) pt[j] = (lo + j * kKvPage) % a.S;  // ring row of the run's first position
        else pt[j] = a.kv_page ? a.kv_page[static_cast<size_t>(b) * a.kv_page_ld + j] : j;
        unmapped |= pt[j] < 0;
    }
    size_t cache_base, page_stride;
    if (RING) {
        cache_base = static_cast<size_t>(kv_ring_row(b, g, a.Hkv, a.S)) * DH;
        page_stride = DH;
    } else {
        cache_base = a.kv_page ? static_cast<size_t>(g) * kKvPage * DH
                               : ((static_cast<size_t>(b) * a.Hkv + g) * a.S + lo) * DH;
        page_stride = static_cast<size_t>(a.kv_page ? a.Hkv : 1) * kKvPage * DH;
    }

    for (int e = threadIdx.x; e < G * DH; e += kAttnThreads) {
        const int gg = e / DH, d = e - gg * DH;
        qs[e] = bf2f(a.q[(static_cast<size_t>(row) * a.H + g * G + gg) * DH + d]);
    }
    if (__syncthreads_or(unmapped)) {  // part of the history is not mapped: attend to nothing, like an idle row
        for (int e = threadIdx.x; e < G * DH; e += kAttnThreads)
            a.out[(static_cast<size_t>(row) * a.H + blockIdx.x * G) * DH + e] = f2bf(0.f);
        return;
    }

    attend<DH, G>(qs, sc, red, a.kcache + cache_base, a.vcache + cache_base, pt, page_stride, L, lcap, scale,
                  a.bf16_math, a.out + (static_cast<size_t>(row) * a.H + g * G) * DH);
}

// ------------------------------------------------------------------------------------------------
// decode-step attention with the qkv GEMM's fix-up in front (see lm_kernels.cuh)
// ------------------------------------------------------------------------------------------------
// SPLIT (attn_decode_split_kernel): a row of more than sp.span positions stops after the front end, its finished q heads
// stored to sp.q for attn_span_kernel; every other row runs the code of SPLIT = false.
template <int DH, int G, bool SPLIT>
__device__ __forceinline__ void attn_decode_body(const AttnDecodeArgs a, const float scale, const int lcap, const AttnSplit sp,
                                                 int* kv_miss) {
    pdl_launch_dependents();
    const int row = blockIdx.y, g = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    extern __shared__ float sm[];
    float* qs = sm;                      // [G][DH]
    float* sc = qs + G * DH;             // [G][lcap]
    float* red = sc + G * lcap;          // [kAttnWarps][G][DH]
    int* pt = reinterpret_cast<int*>(red + kAttnWarps * G * DH);  // this row's pages (attend()); identity if contiguous
    // ---- before the qkv GEMM has finished: this row's page-table entries into registers, and its K/V history towards
    // L2.  The cache lines of positions < pos were written frames ago; the position read here may be one frame stale
    // (it only steers how many entries are loaded early and the prefetch hints; the real one is read after the
    // dependency wait, and the page table does not change during a decode call).  The scores / values loops then find
    // L2 hits instead of paying the HBM latency while the next GEMM's weight prefetch keeps the memory queues full. ----
    const size_t cache_base = a.kv_page ? static_cast<size_t>(g) * kKvPage * DH
                                        : (static_cast<size_t>(a.row_seq[row]) * a.Hkv + g) * a.S * DH;
    const size_t page_stride = static_cast<size_t>(a.kv_page ? a.Hkv : 1) * kKvPage * DH;
    const int* ptab = a.kv_page ? a.kv_page + static_cast<size_t>(a.row_seq[row]) * a.kv_page_ld : nullptr;
    const int pp = min(max(a.row_pos[row], 0), a.S - 1);
    // entry j < npre of the row's page table is held by thread j from here on (one load, off the critical path)
    const int npre = min(min(pp / kKvPage + 2, (a.S + kKvPage - 1) / kKvPage), kAttnThreads);
    const int pg_pre = threadIdx.x < npre ? (ptab ? ptab[threadIdx.x] : static_cast<int>(threadIdx.x)) : -1;
    {
        const int n = min(pp + 1, kAttnPrefetchPos);
        const int lines = n * DH * 2 / 128;  // 128-byte lines of K (and as many of V); a page is whole lines
        constexpr int kLinesPerPage = kKvPage * DH * 2 / 128;
        for (int i = threadIdx.x; i < lines; i += kAttnThreads) {
            const int pg = ptab ? ptab[i / kLinesPerPage] : i / kLinesPerPage;
            if (pg < 0) continue;
            const size_t byte = (cache_base + pg * page_stride) * 2 + static_cast<size_t>(i % kLinesPerPage) * 128;
            prefetch_l2(reinterpret_cast<const char*>(a.kcache) + byte);
            prefetch_l2(reinterpret_cast<const char*>(a.vcache) + byte);
        }
    }
    // what the front end needs besides the GEMM result (static data): requested before the wait as well
    constexpr int HPR = kAttnThreads / DH;   // heads per round
    constexpr int WPH = DH / 32;             // warps per head
    constexpr int NH = G + 2;
    constexpr int NR = (NH + HPR - 1) / HPR;  // rounds: this thread's features, one per round
    const int hsub = threadIdx.x / DH, d = threadIdx.x % DH;
    float bias_r[NR], normw_r[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        const int hh = r * HPR + hsub;
        const int kind = hh < G ? 0 : (hh == G ? 1 : 2);
        const int head = kind == 0 ? g * G + hh : (kind == 1 ? a.H + g : a.H + a.Hkv + g);
        const __nv_bfloat16* nw = kind == 0 ? a.q_norm : (kind == 1 ? a.k_norm : nullptr);
        bias_r[r] = (a.bias != nullptr && hh < NH) ? bf2f(a.bias[head * DH + d]) : 0.f;
        normw_r[r] = (nw != nullptr && hh < NH) ? bf2f(nw[d]) : 0.f;
    }
    pdl_wait();
    __shared__ float wred[NR][kAttnWarps];
    // ---- finish the qkv GEMM for this row's heads: q heads g*G .. g*G+G-1, then k, then v of KV group g.  The
    // partials are requested before the row's position is looked at (they do not depend on it) ----
    const int rpos = a.row_pos[row];
    float vsum[NR];
    {
        int feat[NR];
        bool ok[NR];
#pragma unroll
        for (int r = 0; r < NR; ++r) {
            const int hh = r * HPR + hsub;
            ok[r] = hh < NH;
            const int kind = hh < G ? 0 : (hh == G ? 1 : 2);
            const int head = kind == 0 ? g * G + hh : (kind == 1 ? a.H + g : a.H + a.Hkv + g);
            feat[r] = head * DH + d;
        }
        step_partial_sums<NR>(a.qkv, row, feat, ok, vsum);  // every partial of every round in flight at once
    }
    if (rpos < 0) {  // idle slot parked at position -1: neither the cache nor the output row is touched
        return;
    }
    const int wpos = min(rpos, a.S - 1);
    bool unmapped = false;
    for (int j = threadIdx.x; j <= wpos / kKvPage; j += kAttnThreads) {  // entries the early load did not cover
        pt[j] = j < npre ? pg_pre : (ptab ? ptab[j] : j);  // j < npre: j == threadIdx.x
        unmapped |= pt[j] < 0;
    }
    if (__syncthreads_or(unmapped)) {  // unmapped history: nothing is written, nothing attended, the miss recorded
        if (kv_miss != nullptr && g == 0 && threadIdx.x == 0) {
            int* miss = kv_miss + a.row_seq[row];
            if (*miss == 0) *miss = rpos + 1;
        }
        return;
    }
    const bool split_row = SPLIT && wpos + 1 > sp.span;
    // (cos, sin) of this lane's rotary pair at the row's position: the same for q and k
    const uint32_t cs = *reinterpret_cast<const uint32_t*>(a.freqs + (static_cast<size_t>(wpos) * (DH / 2) + (d >> 1)) * 2);
    // bias, the GEMM output's bf16 rounding, and per-head nn.RMSNorm (fp32 math, weight multiply included, ONE
    // rounding): the sums of squares of all rounds cross the warps behind one barrier
    const bool any_norm = a.q_norm != nullptr || a.k_norm != nullptr;
    float v[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        const int hh = r * HPR + hsub;
        v[r] = 0.f;
        if (hh < NH) {
            v[r] = vsum[r];
            if (a.bias) v[r] += bias_r[r];
            v[r] = rbf(v[r]);
        }
        if (any_norm) {
            const float ws = warp_sum(v[r] * v[r]);
            if (lane == 0) wred[r][warp] = ws;
        }
    }
    if (any_norm) __syncthreads();
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        const int hh = r * HPR + hsub;
        const bool live = hh < NH;
        const int kind = hh < G ? 0 : (hh == G ? 1 : 2);
        const bool normed = kind == 0 ? a.q_norm != nullptr : (kind == 1 ? a.k_norm != nullptr : false);
        float x = v[r];
        if (live && normed) {
            const int w0 = (warp / WPH) * WPH;
            float tot = 0.f;
#pragma unroll
            for (int u = 0; u < WPH; ++u) tot += wred[r][w0 + u];
            const float rinv = rsqrtf(tot / static_cast<float>(DH) + a.eps);
            x = rbf(x * rinv * normw_r[r]);
        }
        if (kind != 2) {
            const float c = bf_lo(cs), sn = bf_hi(cs);
            const float partner = __shfl_xor_sync(0xffffffffu, x, 1);
            x = (lane & 1) ? __fadd_rn(__fmul_rn(x, c), __fmul_rn(partner, sn)) : __fsub_rn(__fmul_rn(x, c), __fmul_rn(partner, sn));
            x = rbf(x);
        }
        if (live) {
            if (kind == 0) {
                qs[hh * DH + d] = x;
                if (split_row) sp.q[(static_cast<size_t>(row) * a.H + g * G + hh) * DH + d] = f2bf(x);  // x is a bf16 value
            } else if (rpos < a.S) {
                __nv_bfloat16* cache = kind == 1 ? a.kcache : a.vcache;
                cache[cache_base + pt[rpos / kKvPage] * page_stride + (rpos % kKvPage) * DH + d] = f2bf(x);
            }
        }
    }
    if (a.kv_only || split_row) return;
    __syncthreads();  // q in shared memory, this row's new K/V visible to the whole CTA

    const int L = wpos + 1;
    attend<DH, G>(qs, sc, red, a.kcache + cache_base, a.vcache + cache_base, pt, page_stride, L, lcap, scale,
                  a.bf16_math, a.out + (static_cast<size_t>(row) * a.H + g * G) * DH);
}

template <int DH, int G>
__global__ void __launch_bounds__(kAttnThreads) attn_decode_kernel(AttnDecodeArgs a, float scale, int lcap,
                                                                   int* kv_miss) {
    attn_decode_body<DH, G, false>(a, scale, lcap, AttnSplit{}, kv_miss);
}

template <int DH, int G>
__global__ void __launch_bounds__(kAttnThreads) attn_decode_split_kernel(AttnDecodeArgs a, AttnSplit sp, float scale,
                                                                         int lcap, int* kv_miss) {
    attn_decode_body<DH, G, true>(a, scale, lcap, sp, kv_miss);
}

// A long row's page-table walk, shared by attn_span_kernel and attn_combine_kernel so that both take the same
// decision: false when any page of positions [0, L) is not mapped (the row then attends to nothing, as in
// attn_decode_kernel). Entries of pages [page0, page0 + npt) go to pt (the identity when the cache is contiguous).
__device__ __forceinline__ bool split_row_pages(const AttnDecodeArgs& a, int row, int L, int page0, int npt, int* pt) {
    const int* ptab = a.kv_page ? a.kv_page + static_cast<size_t>(a.row_seq[row]) * a.kv_page_ld : nullptr;
    bool unmapped = false;
    for (int j = threadIdx.x; j <= (L - 1) / kKvPage; j += kAttnThreads) {
        const int pg = ptab ? ptab[j] : j;
        unmapped |= pg < 0;
        if (j >= page0 && j < page0 + npt) pt[j - page0] = pg;
    }
    return !__syncthreads_or(unmapped);
}

// One span of one long row (see AttnSplit): positions [p0, p0 + n) of KV group g against the row's G query heads. K is
// read once: the span's scores stay in shared memory. Stores acc[G][DH] = sum_p exp(s_p - m) v_p, m = max_p s_p and
// z = sum_p exp(s_p - m) per head. The loops are attend()'s one-pass ones over the span, so every lane and warp sums
// a fixed sequence of terms that depends on the span's positions only.
template <int DH, int G>
__global__ void __launch_bounds__(kAttnThreads) attn_span_kernel(AttnDecodeArgs a, AttnSplit sp, float scale) {
    static_assert(G <= kAttnWarps, "one warp per query head in the softmax");
    pdl_launch_dependents();
    pdl_wait();  // every CTA, the idle ones too: the kernels behind this one count on the whole chain of waits
    const int g = blockIdx.x, row = blockIdx.y, p0 = blockIdx.z * sp.span;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rpos = a.row_pos[row];
    if (rpos < 0) return;  // parked
    const int L = min(rpos, a.S - 1) + 1;
    if (L <= sp.span || p0 >= L) return;  // a short row (attended by the front end), or a span past the row's end
    const int n = min(sp.span, L - p0);
    extern __shared__ float sm[];
    float* qs = sm;                      // [G][DH]
    float* sc = qs + G * DH;             // [G][span]
    float* red = sc + G * sp.span;       // [kAttnWarps][G][DH]
    int* pt = reinterpret_cast<int*>(red + kAttnWarps * G * DH);  // pages of the span
    for (int e = threadIdx.x; e < G * DH; e += kAttnThreads)
        qs[e] = bf2f(sp.q[(static_cast<size_t>(row) * a.H + g * G) * DH + e]);
    if (!split_row_pages(a, row, L, p0 / kKvPage, sp.span / kKvPage, pt)) return;
    const size_t cache_base = a.kv_page ? static_cast<size_t>(g) * kKvPage * DH
                                        : (static_cast<size_t>(a.row_seq[row]) * a.Hkv + g) * a.S * DH;
    const size_t page_stride = static_cast<size_t>(a.kv_page ? a.Hkv : 1) * kKvPage * DH;
    const __nv_bfloat16* kc = a.kcache + cache_base;
    const __nv_bfloat16* vc = a.vcache + cache_base;
    const int lcap = sp.span;

    constexpr int LPR = DH / 8;    // lanes per cache row (16-byte loads)
    constexpr int RPW = 32 / LPR;  // rows per warp iteration
    constexpr int UNR = 4;         // independent 16-byte loads in flight per lane
    constexpr int DPL = DH / 32;   // value dims per lane
    const int sub = lane / LPR, li = lane % LPR;
    auto at = [&](const __nv_bfloat16* base, int p) {  // p relative to the span's first position, a page edge
        return base + static_cast<size_t>(pt[p / kKvPage]) * page_stride + (p % kKvPage) * DH;
    };
    {
        float qr[G][8];
#pragma unroll
        for (int gg = 0; gg < G; ++gg)
#pragma unroll
            for (int e = 0; e < 8; ++e) qr[gg][e] = qs[gg * DH + li * 8 + e];
        for (int pb = warp * RPW * UNR; pb < n; pb += kAttnWarps * RPW * UNR) {
            uint4 u[UNR];
            const __nv_bfloat16* kp = at(kc, pb);  // RPW * UNR positions from a multiple of 8: one page
#pragma unroll
            for (int j = 0; j < UNR; ++j) {
                const int p = pb + j * RPW + sub;
                u[j] = make_uint4(0, 0, 0, 0);
                if (p < n) u[j] = *reinterpret_cast<const uint4*>(kp + (j * RPW + sub) * DH + li * 8);
            }
#pragma unroll
            for (int j = 0; j < UNR; ++j) {
                const int p = pb + j * RPW + sub;
                const bool ok = p < n;
                const float kf[8] = {bf_lo(u[j].x), bf_hi(u[j].x), bf_lo(u[j].y), bf_hi(u[j].y),
                                     bf_lo(u[j].z), bf_hi(u[j].z), bf_lo(u[j].w), bf_hi(u[j].w)};
#pragma unroll
                for (int gg = 0; gg < G; ++gg) {
                    float d = 0.f;
#pragma unroll
                    for (int e = 0; e < 8; ++e) d += qr[gg][e] * kf[e];
#pragma unroll
                    for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
                    if (ok && li == 0) sc[gg * lcap + p] = d * scale;
                }
            }
        }
    }
    __syncthreads();
    float* rec = sp.ws + ((static_cast<size_t>(row) * a.Hkv + g) * gridDim.z + blockIdx.z) * attn_span_floats(G, DH);
    if (warp < G) {
        float* s = sc + warp * lcap;
        float m = -INFINITY, z = 0.f;
        for (int p = lane; p < n; p += 32) m = fmaxf(m, s[p]);
        m = warp_max(m);
        for (int p = lane; p < n; p += 32) {
            const float e = expf(s[p] - m);
            s[p] = e;
            z += e;
        }
        z = warp_sum(z);
        if (lane == 0) {
            rec[G * DH + warp] = m;
            rec[G * DH + G + warp] = z;
        }
    }
    __syncthreads();
    float acc[G][DPL];
#pragma unroll
    for (int gg = 0; gg < G; ++gg)
#pragma unroll
        for (int e = 0; e < DPL; ++e) acc[gg][e] = 0.f;
    for (int pb = warp; pb < n; pb += kAttnWarps * UNR) {
        const __nv_bfloat16* vp = at(vc, pb);  // positions pb + 8 j, inside a run of 32 from a multiple of 32: one page
        float vf[UNR][DPL];
#pragma unroll
        for (int j = 0; j < UNR; ++j) {
            const int p = pb + j * kAttnWarps;
#pragma unroll
            for (int e = 0; e < DPL; ++e) vf[j][e] = 0.f;
            if (p < n) {
                if (DPL == 4) {
                    const uint2 u2 = *reinterpret_cast<const uint2*>(vp + (j * kAttnWarps) * DH + lane * 4);
                    vf[j][0] = bf_lo(u2.x); vf[j][1] = bf_hi(u2.x); vf[j][2 % DPL] = bf_lo(u2.y); vf[j][3 % DPL] = bf_hi(u2.y);
                } else {
                    const uint32_t u1 = *reinterpret_cast<const uint32_t*>(vp + (j * kAttnWarps) * DH + lane * 2);
                    vf[j][0] = bf_lo(u1); vf[j][1] = bf_hi(u1);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < UNR; ++j) {
            const int p = pb + j * kAttnWarps;
            if (p < n) {
#pragma unroll
                for (int gg = 0; gg < G; ++gg) {
                    const float w = sc[gg * lcap + p];
#pragma unroll
                    for (int e = 0; e < DPL; ++e) acc[gg][e] += w * vf[j][e];
                }
            }
        }
    }
#pragma unroll
    for (int gg = 0; gg < G; ++gg)
#pragma unroll
        for (int e = 0; e < DPL; ++e) red[(warp * G + gg) * DH + lane * DPL + e] = acc[gg][e];
    __syncthreads();
    for (int e = threadIdx.x; e < G * DH; e += kAttnThreads) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < kAttnWarps; ++w) s += red[w * G * DH + e];
        rec[e] = s;
    }
}

// Merge of a long row's spans: with M = max_s m_s, out = (sum_s acc_s exp(m_s - M)) / (sum_s z_s exp(m_s - M)), both
// sums in ascending span order, rounded to bf16 once. A kernel of its own rather than the last span CTA to arrive:
// the order of the sum must not depend on which CTA finishes first.
template <int DH, int G>
__global__ void __launch_bounds__(kAttnThreads) attn_combine_kernel(AttnDecodeArgs a, AttnSplit sp) {
    pdl_launch_dependents();
    pdl_wait();  // every CTA: the wo GEMM behind this kernel waits on it for the rows of all three attention kernels
    const int g = blockIdx.x, row = blockIdx.y;
    const int rpos = a.row_pos[row];
    if (rpos < 0) return;
    const int L = min(rpos, a.S - 1) + 1;
    if (L <= sp.span) return;
    if (!split_row_pages(a, row, L, 0, 0, nullptr)) return;
    constexpr int R = attn_span_floats(G, DH);
    const int ns = (L + sp.span - 1) / sp.span, nspans = (sp.bound + sp.span - 1) / sp.span;
    const float* rec = sp.ws + (static_cast<size_t>(row) * a.Hkv + g) * nspans * R;
    __nv_bfloat16* out = a.out + (static_cast<size_t>(row) * a.H + g * G) * DH;
    for (int e = threadIdx.x; e < G * DH; e += kAttnThreads) {
        const int gg = e / DH;
        float M = -INFINITY;
        for (int s = 0; s < ns; ++s) M = fmaxf(M, rec[static_cast<size_t>(s) * R + G * DH + gg]);
        float Z = 0.f, o = 0.f;
        for (int s = 0; s < ns; ++s) {
            const float* r = rec + static_cast<size_t>(s) * R;
            const float w = expf(r[G * DH + gg] - M);
            Z += r[G * DH + G + gg] * w;
            o += r[e] * w;
        }
        out[e] = f2bf(o / Z);
    }
}

// ------------------------------------------------------------------------------------------------
// SwiGLU on a plain fp32 GEMM result (prefill, codec): 4 consecutive features per thread where aligned
// ------------------------------------------------------------------------------------------------
__global__ void swiglu_kernel(SwigluArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.I) return;
    const float* y = a.y + static_cast<size_t>(row) * a.ld;
    const int gi = a.interleaved ? w13_gate_row(i) : i;
    const int ui = a.interleaved ? gi + 16 : a.I + i;
    const float g = rbf(y[gi]), c = rbf(y[ui]);
    const float s = rbf(g / (1.f + expf(-g)));
    a.h[static_cast<size_t>(row) * a.I + i] = f2bf(s * c);
}

__global__ void swiglu4_kernel(SwigluArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.y;
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= a.I) return;
    const float* y = a.y + static_cast<size_t>(row) * a.ld;
    // 4 consecutive h features never straddle a 16-feature interleave group
    const int gi = a.interleaved ? w13_gate_row(i) : i;
    const int ui = a.interleaved ? gi + 16 : a.I + i;
    const float4 g4 = *reinterpret_cast<const float4*>(y + gi);
    const float4 u4 = *reinterpret_cast<const float4*>(y + ui);
    const float gv[4] = {g4.x, g4.y, g4.z, g4.w}, uv[4] = {u4.x, u4.y, u4.z, u4.w};
    float h[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float gg = rbf(gv[c]), cc = rbf(uv[c]);
        const float sl = rbf(gg / (1.f + expf(-gg)));
        h[c] = sl * cc;
    }
    uint2 o;
    o.x = pack_bf2(h[0], h[1]);
    o.y = pack_bf2(h[2], h[3]);
    *reinterpret_cast<uint2*>(a.h + static_cast<size_t>(row) * a.I + i) = o;
}

// ------------------------------------------------------------------------------------------------
// sampling: inference.py:43-93 (logits_to_probs / multinomial_sample_one_no_sync / sample) and the
// slow-token RAS rule inference.py:114-144.
// ------------------------------------------------------------------------------------------------
constexpr int kSampleThreads = 1024;
constexpr int kSelCap = 256;  // ranks materialised for top-k / top-p

__device__ __forceinline__ void philox4x32(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1,
                                           uint32_t c2, uint32_t c3, uint32_t out[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

struct ArgMax {
    float v;
    int i;
};
__device__ __forceinline__ ArgMax better(ArgMax a, ArgMax b) {
    // larger value wins; ties -> smaller index
    if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
    return a;
}
__device__ __forceinline__ ArgMax block_argmax(ArgMax x, ArgMax* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ArgMax y;
        y.v = __shfl_xor_sync(0xffffffffu, x.v, o);
        y.i = __shfl_xor_sync(0xffffffffu, x.i, o);
        x = better(x, y);
    }
    __syncthreads();
    if (lane == 0) red[w] = x;
    __syncthreads();
    if (w == 0) {
        ArgMax t = red[lane];  // kSampleThreads/32 == 32 warps
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            ArgMax y;
            y.v = __shfl_xor_sync(0xffffffffu, t.v, o);
            y.i = __shfl_xor_sync(0xffffffffu, t.i, o);
            t = better(t, y);
        }
        if (lane == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}

// One row of the sampler. FIRST_FRAME (fused admission, slot control only): a row whose slot has produced no frame yet
// samples by the prefill's rule, no RAS substitution and no RAS-window update (inference.py:336-352 samples the first
// frame without previous_tokens); every other row by a.use_ras / a.ras_update as in sample_kernel. The arguments are
// taken by value and each rule is read where it is used, so that sample_kernel compiles to the very instructions it had
// before this template existed.
template <bool FIRST_FRAME>
__device__ __forceinline__ void sample_row(SampleArgs a) {
    __shared__ float lg[kSampleMaxN];
    __shared__ ArgMax red[33];
    __shared__ float fred[33];
    __shared__ float sel_v[kSelCap];
    __shared__ int sel_i[kSelCap];
    __shared__ float sel_cum[kSelCap];
    __shared__ int s_nsel;
    __shared__ int s_choice[2];
    const SlotCtl& ctl = a.ctl;
    const int row = blockIdx.x;
    const int slot = a.row_slot ? a.row_slot[row] : row;
    const int n = a.n;
    if (!slot_live(ctl, slot)) return;  // idle / frozen slot: nothing is sampled, its state stays as it is
    const bool per_slot = ctl.state != nullptr;
    const float temperature = per_slot ? ctl.temperature[slot] : a.temperature;
    const float top_p = per_slot ? ctl.top_p[slot] : a.top_p;
    const int top_k = per_slot ? ctl.top_k[slot] : a.top_k;
    const unsigned long long seed = per_slot ? ctl.seed[slot] : a.seed;
#define FSB_ROW_RULE(flag) (FIRST_FRAME ? ((flag) && ctl.n_out[slot] != 0) : (flag))
    for (int e0 = threadIdx.x; e0 < n; e0 += 4 * kSampleThreads) {
        int feat[4];
        bool ok[4];
        float sum[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            feat[k] = e0 + k * kSampleThreads;
            ok[k] = feat[k] < n;
        }
        step_partial_sums<4>(a.parts, row, feat, ok, sum);  // 32 loads in flight per thread, additions in slot order
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (!ok[k]) continue;
            const float v = rbf(sum[k]);  // F.linear output is a bf16 tensor
            lg[feat[k]] = v;
            if (a.logits_out) a.logits_out[static_cast<size_t>(slot) * n + feat[k]] = v;
        }
    }
    __syncthreads();

    // top_k <= 1 keeps rank 0 only, as the reference's mask does (ranks >= top_k removed, then rank 0 restored): the
    // greedy argmax, and no RAS re-draw, whose top-k cut is the same
    const bool two = a.slow && FSB_ROW_RULE(a.use_ras) && top_k > 1;
    if (top_k <= 1) {
        ArgMax x{-INFINITY, 0x7fffffff};
        for (int e = threadIdx.x; e < n; e += kSampleThreads) x = better(x, ArgMax{lg[e], e});
        x = block_argmax(x, red);
        if (threadIdx.x == 0) s_choice[0] = s_choice[1] = x.i;
        __syncthreads();
    } else {
        // softmax denominator over every candidate (the -inf-biased vocabulary contributes 0)
        float m = -INFINITY;
        for (int e = threadIdx.x; e < n; e += kSampleThreads) m = fmaxf(m, lg[e]);
        m = block_max(m, fred);
        float z = 0.f;
        for (int e = threadIdx.x; e < n; e += kSampleThreads) z += expf(lg[e] - m);
        z = block_sum(z, fred);
        // descending ranks until neither criterion can keep anything further
        const float p_lim = two ? fmaxf(top_p, 0.9f) : top_p;
        int kcap = top_k < n ? top_k : n;
        if (kcap > kSelCap) kcap = kSelCap;
        float cumf = 0.f;  // torch.cumsum over bf16 accumulates in fp32 and rounds each output
        int nsel = 0;
        for (int r = 0; r < kcap; ++r) {
            ArgMax x{-INFINITY, 0x7fffffff};
            for (int e = threadIdx.x; e < n; e += kSampleThreads) x = better(x, ArgMax{lg[e], e});
            x = block_argmax(x, red);
            const float pr = rbf(expf(x.v - m) / z);
            cumf += pr;
            const float cum = rbf(cumf);
            if (threadIdx.x == 0) {
                sel_v[r] = x.v;
                sel_i[r] = x.i;
                sel_cum[r] = cum;
                lg[x.i] = -INFINITY;
            }
            nsel = r + 1;
            __syncthreads();
            if (cum > p_lim) break;
        }
        if (threadIdx.x == 0) s_nsel = nsel;
        __syncthreads();
        // the two draws (normal, RAS high-temperature); warp 0 / warp 1
        const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
        if (w < (two ? 2 : 1)) {
            const float T = w == 0 ? temperature : 1.0f;
            const float tp = w == 0 ? top_p : 0.9f;
            const float Tc = fmaxf(T, 1e-5f);
            // survivors: rank 0 always; rank r kept iff cum[r] <= top_p (and r < top_k, implied)
            int ns = 1;
            while (ns < nsel && !(sel_cum[ns] > tp)) ++ns;
            float mx = -INFINITY;
            for (int r = lane; r < ns; r += 32) mx = fmaxf(mx, rbf(sel_v[r] / Tc));
            mx = warp_max(mx);
            float zz = 0.f;
            for (int r = lane; r < ns; r += 32) zz += expf(rbf(sel_v[r] / Tc) - mx);
            zz = warp_sum(zz);
            // RNG stream: per call (seed, global frame counter, slot) or, with slot control, per request
            // (its own seed and frame index, no slot) so that the draw does not depend on the schedule
            const unsigned long long off =
                per_slot ? static_cast<unsigned long long>(ctl.n_out[slot]) : (a.rng_offset ? *a.rng_offset : 0ull);
            const uint32_t lane_id = per_slot ? 0u : static_cast<uint32_t>(slot);
            const int draw = a.draw_id * 2 + w;
            const float* noise = (a.noise_u != nullptr && slot == 0)
                                     ? a.noise_u + (static_cast<size_t>(off) * a.noise_draws + draw) * a.noise_ld
                                     : nullptr;
            ArgMax best{-INFINITY, 0x7fffffff};
            for (int r = lane; r < ns; r += 32) {
                const float pr = rbf(expf(rbf(sel_v[r] / Tc) - mx) / zz);
                const int e = sel_i[r];
                // torch.argmax returns the first maximum in vocabulary order: ties break on the token id
                const int key = a.slow ? (e < a.n_sem ? a.sem_begin + e : a.im_end_id) : e;
                float score;
                if (noise != nullptr) {
                    const float q = rbf(-logf(noise[e]));  // -log(U) as a bf16 tensor (inference.py:43-46)
                    score = rbf(pr / q);
                } else {
                    uint32_t rnd[4];
                    philox4x32(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32),
                               static_cast<uint32_t>(off), static_cast<uint32_t>(off >> 32), lane_id,
                               static_cast<uint32_t>(draw * kSelCap + r), rnd);
                    const float u = (static_cast<float>(rnd[0] >> 8) + 0.5f) * (1.0f / 16777216.0f);
                    score = pr / -logf(u);
                }
                best = better(best, ArgMax{score, key * kSelCap + r});
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                ArgMax y;
                y.v = __shfl_xor_sync(0xffffffffu, best.v, o);
                y.i = __shfl_xor_sync(0xffffffffu, best.i, o);
                best = better(best, y);
            }
            if (lane == 0) s_choice[w] = sel_i[best.i % kSelCap];
        }
        __syncthreads();
        if (!two && threadIdx.x == 0) s_choice[1] = s_choice[0];
        __syncthreads();
    }

    if (threadIdx.x == 0) {
        int* ct = a.cur_tok + static_cast<size_t>(slot) * (a.num_cb + 1);
        if (a.slow) {
            int e = s_choice[0];
            int tok = e < a.n_sem ? a.sem_begin + e : a.im_end_id;
            if (FSB_ROW_RULE(a.use_ras)) {
                const int eh = s_choice[1];
                const int tok_h = eh < a.n_sem ? a.sem_begin + eh : a.im_end_id;
                bool in_win = false;
                for (int k = 0; k < 10; ++k) in_win |= (a.ras_window[slot * 10 + k] == tok);
                const bool is_sem = tok >= a.sem_begin && tok <= a.sem_begin + a.n_sem - 1;
                if (in_win && is_sem) tok = tok_h;
            }
            int c0 = tok - a.sem_begin;
            c0 = c0 < 0 ? 0 : (c0 > a.codebook_size - 1 ? a.codebook_size - 1 : c0);
            ct[0] = tok;
            ct[1] = c0;
            if (FSB_ROW_RULE(a.ras_update)) {
                for (int k = 0; k < 9; ++k) a.ras_window[slot * 10 + k] = a.ras_window[slot * 10 + k + 1];
                a.ras_window[slot * 10 + 9] = tok;
            }
            if (a.finished && tok == a.im_end_id) a.finished[slot] = 1;
            // the reference's loop tests <|im_end|> from the second frame on (the prefill's token is not
            // tested, inference.py:336-352 then :233)
            if (per_slot && tok == a.im_end_id && ctl.n_out[slot] >= 1) ctl.state[slot] = 3;
        } else {
            ct[a.cb_index + 1] = s_choice[0];
        }
    }
#undef FSB_ROW_RULE
}

__global__ void __launch_bounds__(kSampleThreads) sample_kernel(SampleArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    sample_row<false>(a);
}

__global__ void __launch_bounds__(kSampleThreads) sample_first_frame_kernel(SampleArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    sample_row<true>(a);
}

// ------------------------------------------------------------------------------------------------
// fused admission: stage a deferred prefill's last rows per slot, splice them into the next decode frame
// ------------------------------------------------------------------------------------------------
constexpr int kFirstFrameThreads = 256;

// 16-byte copy of one residual row (D % 8 == 0) and its sums of squares
__device__ __forceinline__ void copy_resid_row(__nv_bfloat16* y, float* y_ssq, const __nv_bfloat16* x,
                                               const float* x_ssq, int D) {
    const uint4* src = reinterpret_cast<const uint4*>(x);
    uint4* dst = reinterpret_cast<uint4*>(y);
    for (int i = threadIdx.x; i < D / 8; i += kFirstFrameThreads) dst[i] = src[i];
    if (threadIdx.x < kSsqRowStride) y_ssq[threadIdx.x] = x_ssq[threadIdx.x];
}

__global__ void __launch_bounds__(kFirstFrameThreads) first_frame_stage_kernel(FirstFrameArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int i = blockIdx.x;
    const int slot = a.slots[i];
    copy_resid_row(a.stage_x + static_cast<size_t>(slot) * a.D, a.stage_ssq + slot * kSsqRowStride,
                   a.x + static_cast<size_t>(i) * a.D, a.ssq + i * kSsqRowStride, a.D);
    if (threadIdx.x == 0) {
        a.stage_pos[slot] = a.row_pos[a.last_rows[i]];
        a.pending[slot] = 1;
        a.pos[slot] = -1;
    }
}

__global__ void __launch_bounds__(kFirstFrameThreads) first_frame_splice_kernel(FirstFrameArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int slot = blockIdx.x;  // decode row r is slot r
    if (a.pending[slot] == 0) return;
    const int s = a.state[slot];
    if (s == 1 || s == 3)
        copy_resid_row(a.x + static_cast<size_t>(slot) * a.D, a.ssq + slot * kSsqRowStride,
                       a.stage_x + static_cast<size_t>(slot) * a.D, a.stage_ssq + slot * kSsqRowStride, a.D);
    __syncthreads();  // every thread has read the flag before it is cleared
    if (threadIdx.x == 0) {
        if (s == 1 || s == 3) a.pos[slot] = a.stage_pos[slot];
        a.pending[slot] = 0;
    }
}

__global__ void frame_end_kernel(FrameEndArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const SlotCtl& ctl = a.ctl;
    const int row = blockIdx.x;
    const int slot = a.row_slot ? a.row_slot[row] : row;
    if (!slot_live(ctl, slot)) return;
    const int f = a.n_out[slot];
    if (threadIdx.x < a.ncols && f < a.T_cap)
        a.out_tokens[(static_cast<size_t>(slot) * a.ncols + threadIdx.x) * a.T_cap + f] =
            a.cur_tok[slot * a.ncols + threadIdx.x];
    __syncthreads();
    if (threadIdx.x == 0) {
        a.n_out[slot] = f + 1;
        bool advance = true;
        if (ctl.state != nullptr && (ctl.state[slot] == 3 || f + 1 >= ctl.limit[slot])) {
            ctl.state[slot] = 2;  // frozen: position and counters stay at the last frame
            advance = false;
        }
        if (a.set_pos_rows)
            a.pos[slot] = a.row_pos_src[a.set_pos_rows[row]] + (advance ? 1 : 0);
        else if (advance)
            a.pos[slot] = a.pos[slot] + 1;
    }
}
// 16-byte copies of positions [0, n_pos) of one (layer, KV head) per CTA row, page by page
__global__ void kv_copy_kernel(uint4* cache, size_t layer16, size_t page16, size_t head16, const int* src_tab,
                               int src0, const int* dst_tab, int dst0, int n16) {
    pdl_launch_dependents();
    pdl_wait();
    const int per_page = static_cast<int>(head16);  // 16-byte units of one (page, head) block
    uint4* base = cache + blockIdx.z * layer16 + blockIdx.y * head16;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n16; e += gridDim.x * blockDim.x) {
        const int j = e / per_page;
        const int sp = src_tab ? src_tab[j] : src0 + j, dp = dst_tab ? dst_tab[j] : dst0 + j;
        if (sp < 0 || dp < 0 || sp == dp) continue;
        const int w = e - j * per_page;
        base[dp * page16 + w] = base[sp * page16 + w];
    }
}

// Blob of one slot's request state (SlotStateArgs): kBlobScalars scalars, the RAS window, cur_tok[ncols], then the
// out_tokens rows [ncols][T_cap] from a 16-byte boundary.
constexpr int kBlobScalars = 10, kBlobRas = 10;
__host__ __device__ inline int blob_head_ints(int ncols) { return (kBlobScalars + kBlobRas + ncols + 3) & ~3; }

// CTA c moves row c of out_tokens (the n_out frames produced so far); CTA 0 also moves the scalars. SAVE: slot ->
// blob, then the slot is parked; otherwise blob -> slot.
template <bool SAVE>
__global__ void slot_state_kernel(SlotStateArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int s = a.slot;
    int* sc = a.blob;
    int* ras = a.blob + kBlobScalars;
    int* ct = ras + kBlobRas;
    const int n = SAVE ? a.n_out[s] : sc[3];
    const size_t row = static_cast<size_t>(blockIdx.x) * a.T_cap;
    int* dev = a.out_tokens + static_cast<size_t>(s) * a.ncols * a.T_cap + row;
    int* sav = a.blob + blob_head_ints(a.ncols) + row;
    for (int f = threadIdx.x; f < n && f < a.T_cap; f += blockDim.x) {
        if (SAVE) sav[f] = dev[f];
        else dev[f] = sav[f];
    }
    if (blockIdx.x != 0) return;
    const int t = threadIdx.x;
    if (t < kBlobRas) {
        if (SAVE) ras[t] = a.ras_window[s * kBlobRas + t];
        else a.ras_window[s * kBlobRas + t] = ras[t];
    }
    if (t >= 32 && t - 32 < a.ncols) {
        if (SAVE) ct[t - 32] = a.cur_tok[s * a.ncols + t - 32];
        else a.cur_tok[s * a.ncols + t - 32] = ct[t - 32];
    }
    if (t != 0) return;
    if (SAVE) {
        const unsigned long long seed = a.seed[s];
        sc[0] = a.state[s]; sc[1] = a.limit[s]; sc[2] = a.top_k[s]; sc[3] = a.n_out[s]; sc[4] = a.pos[s];
        sc[5] = a.finished[s];
        sc[6] = __float_as_int(a.temperature[s]); sc[7] = __float_as_int(a.top_p[s]);
        sc[8] = static_cast<int>(seed & 0xffffffffull); sc[9] = static_cast<int>(seed >> 32);
        a.state[s] = 0;
        a.pos[s] = -1;
    } else {
        a.state[s] = sc[0]; a.limit[s] = sc[1]; a.top_k[s] = sc[2]; a.n_out[s] = sc[3]; a.pos[s] = sc[4];
        a.finished[s] = sc[5];
        a.temperature[s] = __int_as_float(sc[6]); a.top_p[s] = __int_as_float(sc[7]);
        a.seed[s] = static_cast<unsigned long long>(static_cast<unsigned int>(sc[8])) |
                    (static_cast<unsigned long long>(static_cast<unsigned int>(sc[9])) << 32);
    }
}

__global__ void step_inc_kernel(unsigned long long* step) {
    pdl_launch_dependents();
    pdl_wait();
    *step += 1;
}

}  // namespace

int launch_embed(const EmbedArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    FSB_CHECK(a.D % 4 == 0 && a.D <= kSsqTile * kSsqRowStride, "embed: D=%d unsupported", a.D);
    FSB_LAUNCH(embed_kernel, dim3(a.rows), dim3(kRowThreads), 0, st, a, sqrtf(static_cast<float>(a.C + 1)));
    return 0;
}

int launch_rows(const RowsArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    FSB_CHECK(a.D % 4 == 0 && a.D <= kSsqTile * kSsqRowStride, "rows: D=%d unsupported", a.D);
    FSB_CHECK(a.norm_w == nullptr || a.ssq_in != nullptr, "rows: the norm needs the input's sum of squares");
    FSB_LAUNCH(rows_kernel, dim3(a.rows), dim3(kRowThreads), 0, st, a);
    return 0;
}

int launch_resid_norm(const ResidNormArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    FSB_CHECK(a.D <= kRnThreads * kRnMaxPer, "resid_norm: D=%d too large", a.D);
    const bool vec = (a.D & 3) == 0 && (a.y == nullptr || ((a.ld & 3) == 0 && (reinterpret_cast<uintptr_t>(a.y) & 15) == 0));
    if (vec) FSB_LAUNCH(resid_norm4_kernel, dim3(a.rows), dim3(kRn4Threads), 0, st, a);
    else FSB_LAUNCH(resid_norm_kernel, dim3(a.rows), dim3(kRnThreads), 0, st, a);
    return 0;
}

int launch_qkv_prep(const QkvPrepArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    FSB_CHECK(a.Dh % 64 == 0 && a.Dh <= 256, "qkv_prep: head_dim %d unsupported", a.Dh);
    FSB_CHECK((a.ld & 1) == 0 && (reinterpret_cast<uintptr_t>(a.y) & 7) == 0, "qkv_prep: misaligned GEMM result");
    if (a.ring) {
        FSB_CHECK(a.kv_page == nullptr && a.S > 0 && a.S % kKvPage == 0 && (a.Dh == 64 || a.Dh == 128),
                  "qkv_prep: a ring cache needs S a multiple of %d (S=%d), head_dim 64 or 128 and no page table", kKvPage,
                  a.S);
        if (a.Dh == 64) FSB_LAUNCH((qkv_prep_row_kernel<64, true>), dim3(a.rows), dim3(kQkvRowThreads), 0, st, a);
        else FSB_LAUNCH((qkv_prep_row_kernel<128, true>), dim3(a.rows), dim3(kQkvRowThreads), 0, st, a);
        return 0;
    }
    if (a.Dh == 64) FSB_LAUNCH((qkv_prep_row_kernel<64, false>), dim3(a.rows), dim3(kQkvRowThreads), 0, st, a);
    else if (a.Dh == 128) FSB_LAUNCH((qkv_prep_row_kernel<128, false>), dim3(a.rows), dim3(kQkvRowThreads), 0, st, a);
    else FSB_LAUNCH(qkv_prep_kernel, dim3(a.rows, a.H + 2 * a.Hkv), dim3(a.Dh / 2), 0, st, a);
    return 0;
}

// Score-buffer positions per head for a context bound of `need`: rounded up to a multiple of 32 and cut to what fits
// 200 KB of shared memory (a longer context is walked in chunks, see attend()).  g_attn_chunk (tests) forces a chunk.
static int g_attn_chunk = 0;
static bool g_attn_per_row = false;  // tests: launch_attn uses the per-row kernel (the decode kernel's attention core)
void attn_set_score_chunk(int positions) { g_attn_chunk = positions > 0 ? (positions + 31) / 32 * 32 : 0; }
void attn_force_per_row(bool on) { g_attn_per_row = on; }
// `pages`: page-table entries of one row kept in shared memory
template <int DH, int G>
static size_t attn_smem_bytes(int lcap, int pages) {
    return (static_cast<size_t>(G) * DH + static_cast<size_t>(G) * lcap + static_cast<size_t>(kAttnWarps) * G * DH) *
               sizeof(float) + static_cast<size_t>(pages) * sizeof(int);
}
template <int DH, int G>
static int attn_score_chunk(int need, int pages) {
    int lcap = (need + 31) / 32 * 32;
    const int fit = static_cast<int>((200 * 1024 - attn_smem_bytes<DH, G>(0, pages)) / (sizeof(float) * G)) / 32 * 32;
    if (lcap > fit) lcap = fit;
    if (g_attn_chunk > 0 && g_attn_chunk < lcap) lcap = g_attn_chunk;
    return lcap;
}

template <int DH, int G>
static int launch_attn_t(const AttnArgs& a, cudaStream_t st) {
    int lcap = a.window > 0 && a.window < a.S ? a.window : a.S;
    if (a.lcap > 0 && a.lcap < lcap) lcap = a.lcap;
    const int pages = cdiv(a.S, kKvPage);  // page-table entries of one row (the identity when contiguous)
    lcap = attn_score_chunk<DH, G>(lcap, pages);
    const size_t smem = attn_smem_bytes<DH, G>(lcap, pages);
    const float scale = 1.0f / sqrtf(static_cast<float>(DH));
    if (a.ring) FSB_LAUNCH((attn_kernel<DH, G, true>), dim3(a.Hkv, a.rows), dim3(kAttnThreads), smem, st, a, scale, lcap);
    else FSB_LAUNCH((attn_kernel<DH, G, false>), dim3(a.Hkv, a.rows), dim3(kAttnThreads), smem, st, a, scale, lcap);
    return 0;
}

int attn_init() {
    static bool done = false;
    if (done) return 0;
#define FSB_ATTN_ATTR(DH_, G_) \
    FSB_CUDA(cudaFuncSetAttribute(attn_kernel<DH_, G_, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); \
    FSB_CUDA(cudaFuncSetAttribute(attn_kernel<DH_, G_, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); \
    FSB_CUDA(cudaFuncSetAttribute(attn_decode_kernel<DH_, G_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); \
    FSB_CUDA(cudaFuncSetAttribute(attn_decode_split_kernel<DH_, G_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); \
    FSB_CUDA(cudaFuncSetAttribute(attn_span_kernel<DH_, G_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    FSB_ATTN_ATTR(128, 1) FSB_ATTN_ATTR(128, 2) FSB_ATTN_ATTR(128, 4) FSB_ATTN_ATTR(128, 8)
    FSB_ATTN_ATTR(64, 1) FSB_ATTN_ATTR(64, 2) FSB_ATTN_ATTR(64, 4) FSB_ATTN_ATTR(64, 8)
#undef FSB_ATTN_ATTR
    done = true;
    return 0;
}

template <int DH, int G>
static int launch_attn_decode_t(const AttnDecodeArgs& a, cudaStream_t st, int* kv_miss) {
    int lcap = a.S;
    if (a.lcap > 0 && a.lcap < lcap) lcap = a.lcap;
    const int pages = cdiv(a.S, kKvPage);  // page-table entries of one row (the identity when contiguous)
    lcap = attn_score_chunk<DH, G>(lcap, pages);
    const size_t smem = attn_smem_bytes<DH, G>(lcap, pages);
    const float scale = 1.0f / sqrtf(static_cast<float>(DH));
    FSB_LAUNCH((attn_decode_kernel<DH, G>), dim3(a.Hkv, a.rows), dim3(kAttnThreads), smem, st, a, scale, lcap, kv_miss);
    return 0;
}

int launch_attn_decode(const AttnDecodeArgs& a, cudaStream_t st, int* kv_miss) {
    if (a.rows <= 0) return 0;
    const int G = a.H / a.Hkv;
    FSB_CHECK(a.H % a.Hkv == 0, "attention: H %% Hkv != 0");
#define FSB_ATTN_CASE(DH_, G_) \
    if (a.Dh == DH_ && G == G_) return launch_attn_decode_t<DH_, G_>(a, st, kv_miss);
    FSB_ATTN_CASE(128, 1) FSB_ATTN_CASE(128, 2) FSB_ATTN_CASE(128, 4) FSB_ATTN_CASE(128, 8)
    FSB_ATTN_CASE(64, 1) FSB_ATTN_CASE(64, 2) FSB_ATTN_CASE(64, 4) FSB_ATTN_CASE(64, 8)
#undef FSB_ATTN_CASE
    set_error("attention: unsupported head_dim=%d group=%d", a.Dh, G);
    return 1;
}

// shared memory of attn_span_kernel for a span of `span` positions
template <int DH, int G>
static size_t attn_span_smem_bytes(int span) {
    return attn_smem_bytes<DH, G>(span, span / kKvPage);
}

template <int DH, int G>
static int launch_attn_decode_split_t(const AttnDecodeArgs& a, const AttnSplit& sp, cudaStream_t st, int* kv_miss) {
    int lcap = a.S;
    if (a.lcap > 0 && a.lcap < lcap) lcap = a.lcap;
    const int pages = cdiv(a.S, kKvPage);
    lcap = attn_score_chunk<DH, G>(lcap, pages);
    const float scale = 1.0f / sqrtf(static_cast<float>(DH));
    FSB_LAUNCH((attn_decode_split_kernel<DH, G>), dim3(a.Hkv, a.rows), dim3(kAttnThreads),
               (attn_smem_bytes<DH, G>(lcap, pages)), st, a, sp, scale, lcap, kv_miss);
    if (a.kv_only) return 0;
    FSB_LAUNCH((attn_span_kernel<DH, G>), dim3(a.Hkv, a.rows, cdiv(sp.bound, sp.span)), dim3(kAttnThreads),
               (attn_span_smem_bytes<DH, G>(sp.span)), st, a, sp, scale);
    FSB_LAUNCH((attn_combine_kernel<DH, G>), dim3(a.Hkv, a.rows), dim3(kAttnThreads), 0, st, a, sp);
    return 0;
}

int attn_split_max_span(int H, int Hkv, int Dh) {
    if (Hkv <= 0 || H % Hkv != 0) return 0;
    const int G = H / Hkv;
#define FSB_ATTN_CASE(DH_, G_)                                                                                \
    if (Dh == DH_ && G == G_)                                                                                 \
        return static_cast<int>((200 * 1024 - attn_span_smem_bytes<DH_, G_>(0)) / (sizeof(float) * G_ + 1)) / \
               kKvPage * kKvPage;
    FSB_ATTN_CASE(128, 1) FSB_ATTN_CASE(128, 2) FSB_ATTN_CASE(128, 4) FSB_ATTN_CASE(128, 8)
    FSB_ATTN_CASE(64, 1) FSB_ATTN_CASE(64, 2) FSB_ATTN_CASE(64, 4) FSB_ATTN_CASE(64, 8)
#undef FSB_ATTN_CASE
    return 0;
}

int launch_attn_decode_split(const AttnDecodeArgs& a, const AttnSplit& sp, cudaStream_t st, int* kv_miss) {
    if (a.rows <= 0) return 0;
    const int G = a.H / a.Hkv;
    FSB_CHECK(a.H % a.Hkv == 0, "attention: H %% Hkv != 0");
    FSB_CHECK(a.bf16_math == 0, "attention: the split runs the fp32 attention only");
    FSB_CHECK(sp.span > 0 && sp.span % kKvPage == 0 && sp.span <= attn_split_max_span(a.H, a.Hkv, a.Dh),
              "attention: a span of %d positions is not a multiple of %d in [%d, %d]", sp.span, kKvPage, kKvPage,
              attn_split_max_span(a.H, a.Hkv, a.Dh));
    FSB_CHECK(sp.bound > 0 && cdiv(sp.bound, sp.span) <= 65535, "attention: %d spans", cdiv(sp.bound, sp.span));
#define FSB_ATTN_CASE(DH_, G_) \
    if (a.Dh == DH_ && G == G_) return launch_attn_decode_split_t<DH_, G_>(a, sp, st, kv_miss);
    FSB_ATTN_CASE(128, 1) FSB_ATTN_CASE(128, 2) FSB_ATTN_CASE(128, 4) FSB_ATTN_CASE(128, 8)
    FSB_ATTN_CASE(64, 1) FSB_ATTN_CASE(64, 2) FSB_ATTN_CASE(64, 4) FSB_ATTN_CASE(64, 8)
#undef FSB_ATTN_CASE
    set_error("attention: unsupported head_dim=%d group=%d", a.Dh, G);
    return 1;
}

int launch_attn(const AttnArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    FSB_CHECK(a.kv_page == nullptr || a.window <= 0, "attention: a paged KV cache takes no window");
    FSB_CHECK(!a.ring || (a.kv_page == nullptr && a.S > 0 && a.S % kKvPage == 0 && a.window > 0 && a.window < a.S),
              "attention: a ring cache needs S a multiple of %d (S=%d) and 0 < window < S (window=%d)", kKvPage, a.S,
              a.window);
    // one kernel whatever the number of rows: a sequence must get the same bits alone, in a batch or in pieces
    if (!g_attn_per_row && attn_tile_supported(a)) return launch_attn_tile(a, st);
    const int G = a.H / a.Hkv;
    FSB_CHECK(a.H % a.Hkv == 0, "attention: H %% Hkv != 0");
#define FSB_ATTN_CASE(DH_, G_) \
    if (a.Dh == DH_ && G == G_) return launch_attn_t<DH_, G_>(a, st);
    FSB_ATTN_CASE(128, 1) FSB_ATTN_CASE(128, 2) FSB_ATTN_CASE(128, 4) FSB_ATTN_CASE(128, 8)
    FSB_ATTN_CASE(64, 1) FSB_ATTN_CASE(64, 2) FSB_ATTN_CASE(64, 4) FSB_ATTN_CASE(64, 8)
#undef FSB_ATTN_CASE
    set_error("attention: unsupported head_dim=%d group=%d", a.Dh, G);
    return 1;
}

int launch_swiglu(const SwigluArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    const bool vec = (a.I & 3) == 0 && (a.ld & 3) == 0 && (reinterpret_cast<uintptr_t>(a.y) & 15) == 0;
    if (vec) FSB_LAUNCH(swiglu4_kernel, dim3(cdiv(a.I, 1024), a.rows), dim3(256), 0, st, a);
    else FSB_LAUNCH(swiglu_kernel, dim3(cdiv(a.I, 256), a.rows), dim3(256), 0, st, a);
    return 0;
}

int launch_sample(const SampleArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    FSB_CHECK(a.n > 0 && a.n <= kSampleMaxN, "sample: n=%d out of range", a.n);
    FSB_LAUNCH(sample_kernel, dim3(a.rows), dim3(kSampleThreads), 0, st, a);
    return 0;
}

int launch_sample_first_frame(const SampleArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    FSB_CHECK(a.n > 0 && a.n <= kSampleMaxN, "sample: n=%d out of range", a.n);
    FSB_CHECK(a.ctl.state != nullptr && a.slow, "sample: the first-frame rule needs slot control and the slow head");
    FSB_LAUNCH(sample_first_frame_kernel, dim3(a.rows), dim3(kSampleThreads), 0, st, a);
    return 0;
}

int launch_first_frame_stage(const FirstFrameArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    FSB_CHECK(a.D % 8 == 0 && a.D <= kSsqTile * kSsqRowStride, "first_frame_stage: D=%d unsupported", a.D);
    FSB_LAUNCH(first_frame_stage_kernel, dim3(a.rows), dim3(kFirstFrameThreads), 0, st, a);
    return 0;
}

int launch_first_frame_splice(const FirstFrameArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return 0;
    FSB_CHECK(a.D % 8 == 0 && a.D <= kSsqTile * kSsqRowStride, "first_frame_splice: D=%d unsupported", a.D);
    FSB_LAUNCH(first_frame_splice_kernel, dim3(a.rows), dim3(kFirstFrameThreads), 0, st, a);
    return 0;
}

int launch_kv_copy(__nv_bfloat16* cache, int layers, int n_pages, int Hkv, int Dh, const int* src_tab, int src0,
                   const int* dst_tab, int dst0, int n_pos, cudaStream_t st) {
    if (n_pos <= 0) return 0;
    FSB_CHECK(Dh % 8 == 0, "kv_copy: head_dim %d", Dh);
    FSB_CHECK(src_tab != nullptr || (src0 >= 0 && src0 < n_pages && dst0 >= 0 && dst0 < n_pages && n_pos <= kKvPage),
              "kv_copy: page %d -> %d (%d positions) outside the pool of %d pages", src0, dst0, n_pos, n_pages);
    const size_t head16 = static_cast<size_t>(kKvPage) * Dh / 8, page16 = head16 * Hkv, layer16 = page16 * n_pages;
    const int n16 = n_pos * (Dh / 8);
    FSB_LAUNCH(kv_copy_kernel, dim3(cdiv(n16, 256 * 4), Hkv, layers), dim3(256), 0, st,
               reinterpret_cast<uint4*>(cache), layer16, page16, head16, src_tab, src0, dst_tab, dst0, n16);
    return 0;
}

size_t slot_blob_ints(int ncols, int T_cap) {
    return static_cast<size_t>(blob_head_ints(ncols)) + static_cast<size_t>(ncols) * T_cap;
}

int launch_slot_save(const SlotStateArgs& a, cudaStream_t st) {
    FSB_CHECK(a.ncols >= 1 && a.ncols <= 224, "slot_save: %d token rows unsupported", a.ncols);
    FSB_LAUNCH(slot_state_kernel<true>, dim3(a.ncols), dim3(256), 0, st, a);
    return 0;
}

int launch_slot_restore(const SlotStateArgs& a, cudaStream_t st) {
    FSB_CHECK(a.ncols >= 1 && a.ncols <= 224, "slot_restore: %d token rows unsupported", a.ncols);
    FSB_LAUNCH(slot_state_kernel<false>, dim3(a.ncols), dim3(256), 0, st, a);
    return 0;
}

int launch_frame_end(const FrameEndArgs& a, cudaStream_t st) {
    FSB_LAUNCH(frame_end_kernel, dim3(a.rows), dim3(32), 0, st, a);
    FSB_LAUNCH(step_inc_kernel, dim3(1), dim3(1), 0, st, a.step);
    return 0;
}

}  // namespace fsb
