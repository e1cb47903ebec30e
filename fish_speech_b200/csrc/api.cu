// Library-level C-ABI entry points + the unit-test hooks declared in include/fishb200.h.
#include "../../include/fishb200.h"
#include <algorithm>
#include <vector>

#include "gemm_tc.cuh"
#include "lm_gemm.cuh"
#include "lm_kernels.cuh"

using namespace fsb;

extern "C" {

const char* fsb_last_error(void) { return get_error(); }
long long fsb_launch_count(void) { return g_launch_count; }

int fsb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    cudaDeviceProp prop;
    FSB_CUDA(cudaGetDevice(&dev));
    FSB_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return 0;
}

int fsb_memcpy_d2h(void* h_dst, const void* d_src, size_t bytes, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CUDA(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, st));
    FSB_CUDA(cudaStreamSynchronize(st));
    return 0;
}
int fsb_memcpy_h2d(void* d_dst, const void* h_src, size_t bytes, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CUDA(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, st));
    FSB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

// Reduce stream-K partial sums: out[j][i] = sum_s ws[s][j][i]
static __global__ void reduce_parts_kernel(const float* ws, long long slot_stride, const int* nparts,
                                           float* out, int m, int n) {
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
    if (i >= m || j >= n) return;
    const int np = nparts[i >> 7];
    float s = 0.f;
    for (int q = 0; q < np; ++q) s += ws[q * slot_stride + static_cast<long long>(j) * m + i];
    out[static_cast<long long>(j) * m + i] = s;
}

int fsb_op_gemm(const void* d_a, const void* d_b, float* d_out, int m, int n, int k, int bn,
                int streamk_ctas, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    GemmPlan plan;
    memset(&plan, 0, sizeof(plan));
    GemmOperand A{reinterpret_cast<const __nv_bfloat16*>(d_a), k, m, 1, k, static_cast<long long>(m) * k};
    GemmOperand B{reinterpret_cast<const __nv_bfloat16*>(d_b), k, n, 1, k, static_cast<long long>(n) * k};
    const int kblocks = cdiv(k, 64);
    plan.p.kb_per_tap = kblocks;
    plan.p.num_taps = 1;
    plan.p.rows_i = m;
    plan.p.rows_j = n;
    const int tiles_i = cdiv(m, 128), tiles_j = cdiv(n, bn);
    FSB_TRY(gemm_plan_init(&plan, A, B, bn, 6, tiles_i, tiles_j, 1));
    float* ws = nullptr;
    if (streamk_ctas > 0) {
        FSB_CHECK(tiles_j == 1, "stream-K hook needs n <= bn");
        FSB_TRY(gemm_plan_streamk(&plan, tiles_i, kblocks, streamk_ctas));
        const size_t slot = static_cast<size_t>(n) * m;
        FSB_CUDA(cudaMalloc(&ws, slot * plan.max_parts * sizeof(float)));
        plan.p.mode = 0;
        plan.p.ws = ws;
        plan.p.ws_ld = m;
        plan.p.ws_slot_stride = static_cast<long long>(slot);
        int rc = gemm_launch(plan, st);
        if (rc == 0) {
            reduce_parts_kernel<<<dim3(cdiv(m, 256), n), 256, 0, st>>>(ws, plan.p.ws_slot_stride,
                                                                       plan.nparts_dev, d_out, m, n);
            if (cudaGetLastError() != cudaSuccess) rc = 1;
        }
        cudaError_t e = cudaStreamSynchronize(st);
        cudaFree(ws);
        gemm_plan_free(&plan);
        FSB_CHECK(rc == 0, "%s", get_error());
        FSB_CUDA(e);
        return 0;
    }
    // direct fp32 epilogue: out[j*m + i]
    plan.p.mode = 1;
    plan.p.out0 = d_out;
    plan.p.out_f32 = 1;
    plan.p.o_zs = 0;
    plan.p.o_is = 1;
    plan.p.o_js = m;
    plan.p.chan_on_i = 1;
    int rc = gemm_launch(plan, st);
    cudaError_t e = cudaStreamSynchronize(st);
    gemm_plan_free(&plan);
    if (rc != 0) return rc;
    FSB_CUDA(e);
    return 0;
}

// out[j][i] = the step GEMM's partials summed by both consumer helpers; an element where the two disagree in any bit is
// stored as NaN (step_partial_sums promises the same sums as step_partial_sum)
static __global__ void step_sum_kernel(StepPartials P, int rows, float* out) {
    constexpr int N = 4;
    pdl_wait();
    const int f0 = (blockIdx.x * blockDim.x + threadIdx.x) * N, row = blockIdx.y;
    if (f0 >= P.n_out || row >= rows) return;
    int feat[N];
    bool ok[N];
    float s[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
        feat[k] = f0 + k;
        ok[k] = f0 + k < P.n_out;
    }
    step_partial_sums<N>(P, row, feat, ok, s);
#pragma unroll
    for (int k = 0; k < N; ++k) {
        if (!ok[k]) continue;
        const float one = step_partial_sum(P, row, feat[k]);
        const bool same = __float_as_uint(one) == __float_as_uint(s[k]);
        out[static_cast<size_t>(row) * P.n_out + feat[k]] = same ? s[k] : __uint_as_float(0x7fc00000u);
    }
}

int fsb_op_step_gemm_tile(const void* d_w, int n_out, int K, const void* d_x, int row_tile, int rows,
                          const void* d_norm_w, const float* d_x_ssq, float eps, int num_ctas, int stages, float* d_out,
                          int* info, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FSB_CHECK(d_w && d_x && d_out, "step GEMM hook: null operand");
    FSB_CHECK(row_tile == kStepRows || row_tile == kStepRowsMax, "step GEMM hook: row_tile=%d is not %d or %d",
              row_tile, kStepRows, kStepRowsMax);
    FSB_CHECK(rows >= 1 && rows <= row_tile, "step GEMM hook: rows=%d outside [1, %d]", rows, row_tile);
    FSB_CHECK(n_out >= 1 && K >= 1, "step GEMM hook: empty GEMM (n_out=%d, K=%d)", n_out, K);
    FSB_CHECK(num_ctas >= 1 && stages >= 2, "step GEMM hook: num_ctas=%d, stages=%d", num_ctas, stages);
    const bool norm = d_norm_w != nullptr;
    FSB_CHECK(!norm || (d_x_ssq != nullptr && K <= kSsqStride * 128),
              "step GEMM hook: normalise-on-load needs the sums of squares and K <= %d", kSsqStride * 128);
    StepGemmPlan plan;
    // the workspace is sized from the plan's own slot count, so the bound check of step_plan_init is not needed here
    if (step_plan_init(&plan, reinterpret_cast<const __nv_bfloat16*>(d_w), n_out, K,
                       reinterpret_cast<const __nv_bfloat16*>(d_x), norm, row_tile, num_ctas, stages, nullptr,
                       SIZE_MAX) != 0) {
        step_plan_free(&plan);
        return 1;
    }
    const size_t ws_floats = static_cast<size_t>(plan.max_parts) * plan.p.tiles * 128 * row_tile;
    float* ws = nullptr;
    cudaError_t e = cudaMalloc(&ws, ws_floats * sizeof(float));
    int rc = e == cudaSuccess ? 0 : 1;
    if (rc) set_error("step GEMM hook: cudaMalloc: %s", cudaGetErrorString(e));
    if (rc == 0 && info) {
        // what the plan really schedules, read back from the schedule the kernel consumes
        const int ctas = static_cast<int>(plan.grid.x);
        std::vector<int> cta_items(ctas + 1);
        std::vector<int4> items;
        e = cudaMemcpy(cta_items.data(), plan.cta_items_dev, cta_items.size() * sizeof(int), cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) {
            items.resize(cta_items[ctas]);
            e = cudaMemcpy(items.data(), plan.sched_dev, items.size() * sizeof(int4), cudaMemcpyDeviceToHost);
        }
        if (e != cudaSuccess) {
            set_error("step GEMM hook: schedule read-back: %s", cudaGetErrorString(e));
            rc = 1;
        }
        int max_units = 0, max_items = 0;
        for (int c = 0; rc == 0 && c < ctas; ++c) {
            int units = 0;
            for (int n = cta_items[c]; n < cta_items[c + 1]; ++n) units += items[n].z - items[n].y;
            max_units = std::max(max_units, units);
            max_items = std::max(max_items, cta_items[c + 1] - cta_items[c]);
        }
        info[0] = ctas;
        info[1] = plan.p.stages;
        info[2] = plan.max_parts;
        info[3] = max_units;
        info[4] = max_items;
    }
    if (rc == 0) {
        plan.p.ws = ws;
        if (norm) {
            plan.p.x_ssq = d_x_ssq;
            plan.p.norm_w = reinterpret_cast<const __nv_bfloat16*>(d_norm_w);
            plan.p.x_nt = cdiv(K, 128);
            plan.p.eps = eps;
        }
        // all-ones bits = NaN: a slot the consumers add without any CTA having written it shows up in the result
        e = cudaMemsetAsync(ws, 0xff, ws_floats * sizeof(float), st);
        if (e != cudaSuccess) {
            set_error("step GEMM hook: cudaMemsetAsync: %s", cudaGetErrorString(e));
            rc = 1;
        }
    }
    if (rc == 0) rc = step_gemm_launch(plan, rows, st);
    if (rc == 0) {
        const StepPartials P = step_plan_partials(plan);
        step_sum_kernel<<<dim3(cdiv(cdiv(n_out, 4), 128), rows), 128, 0, st>>>(P, rows, d_out);
        e = cudaGetLastError();
        if (e != cudaSuccess) {
            set_error("step GEMM hook: partial sums: %s", cudaGetErrorString(e));
            rc = 1;
        }
    }
    e = cudaStreamSynchronize(st);
    if (ws) cudaFree(ws);
    step_plan_free(&plan);
    if (rc != 0) return rc;
    FSB_CUDA(e);
    return 0;
}

int fsb_op_step_gemm(const void* d_w, int n_out, int K, const void* d_x, int rows, const void* d_norm_w,
                     const float* d_x_ssq, float eps, int num_ctas, int stages, float* d_out, int* info, void* stream) {
    FSB_CHECK(rows >= 1 && rows <= kStepRows, "step GEMM hook: rows=%d outside [1, %d]", rows, kStepRows);
    return fsb_op_step_gemm_tile(d_w, n_out, K, d_x, kStepRows, rows, d_norm_w, d_x_ssq, eps, num_ctas, stages, d_out,
                                 info, stream);
}

}  // extern "C"
