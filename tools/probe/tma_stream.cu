// Probe: how fast can TMA stream a weight matrix into a shared-memory ring, as a function of its HBM layout?
//   layout 0: row-major [N][K] bf16, box {64 k, 128 rows}: 128 segments of 128 B, K*2 bytes apart (checkpoint layout)
//   layout 1: pre-tiled: every (128-row tile, 64-col k-block) is one contiguous 16 KB block
// Same bytes, same request size, same ring; only the DRAM access pattern differs.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../fish_speech_b200/csrc/gemm_tc.cuh"
using namespace fsb;

__global__ void __launch_bounds__(64, 2) stream_kernel(const __grid_constant__ CUtensorMap tm, int tiles, int kblocks, int stages,
                                                       int tiled, unsigned long long hint, unsigned* sink) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const uint32_t full0 = base + stages * 16384u, empty0 = full0 + 8u * stages;
    const long long U = static_cast<long long>(tiles) * kblocks;
    const long long u0 = U * blockIdx.x / gridDim.x, u1 = U * (blockIdx.x + 1) / gridDim.x;
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) { mbar_init(full0 + 8u * s, 1); mbar_init(empty0 + 8u * s, 1); }
        fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int it = 0;
        for (long long u = u0; u < u1; ++u, ++it) {
            const int s = it % stages; const uint32_t ph = (it / stages) & 1u;
            mbar_wait(empty0 + 8u * s, ph ^ 1u);
            mbar_expect_tx(full0 + 8u * s, 16384);
            const int t = static_cast<int>(u / kblocks), kb = static_cast<int>(u % kblocks);
            if (tiled) tma_load_3d(base + s * 16384u, &tm, full0 + 8u * s, 0, static_cast<int>(u) * 128, 0, hint);
            else tma_load_3d(base + s * 16384u, &tm, full0 + 8u * s, kb * 64, t * 128, 0, hint);
        }
    } else if (threadIdx.x == 32) {
        int it = 0; unsigned acc = 0;
        for (long long u = u0; u < u1; ++u, ++it) {
            const int s = it % stages; const uint32_t ph = (it / stages) & 1u;
            mbar_wait(full0 + 8u * s, ph);
            acc += *reinterpret_cast<volatile unsigned*>(smem_raw + (base - raw) + s * 16384);
            mbar_arrive(empty0 + 8u * s);
        }
        if (acc == 0x12345678u) *sink = acc;
    }
}

int main(int argc, char** argv) {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int N = 19456, K = 2560;  // w1|w3 of one S2-Pro layer: 99.6 MB
    const int tiles = N / 128, kblocks = K / 64;
    const int layers = 12;  // rotate over distinct matrices >> L2
    __nv_bfloat16* w;
    const size_t per = static_cast<size_t>(N) * K;
    cudaMalloc(&w, per * 2 * layers);
    cudaMemset(w, 1, per * 2 * layers);
    unsigned* sink; cudaMalloc(&sink, 4);
    cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int tiled = 0; tiled < 2; ++tiled)
        for (int per_sm : {1, 2})
            for (int stages : {3, 4, 5, 6})
                for (int hintsel = 0; hintsel < 2; ++hintsel) {
                    if (per_sm == 2 && stages > 6) continue;
                    std::vector<CUtensorMap> tms(layers);
                    for (int l = 0; l < layers; ++l) {
                        GemmOperand A = tiled ? GemmOperand{w + per * l, 64, static_cast<long long>(tiles) * kblocks * 128, 1, 64, static_cast<long long>(per)}
                                              : GemmOperand{w + per * l, K, N, 1, K, static_cast<long long>(per)};
                        if (gemm_make_tmap(&tms[l], A, 128) != 0) { printf("tmap failed: %s\n", get_error()); return 1; }
                    }
                    const size_t smem = 1024 + stages * 16384 + 16 * stages + 64;
                    const unsigned long long hint = hintsel ? kEvictFirst : kEvictNormal;
                    for (int l = 0; l < layers; ++l) stream_kernel<<<sms * per_sm, 64, smem>>>(tms[l], tiles, kblocks, stages, tiled, hint, sink);
                    cudaEventRecord(e0);
                    const int reps = 3;
                    for (int r = 0; r < reps; ++r)
                        for (int l = 0; l < layers; ++l) stream_kernel<<<sms * per_sm, 64, smem>>>(tms[l], tiles, kblocks, stages, tiled, hint, sink);
                    cudaEventRecord(e1);
                    cudaError_t err = cudaDeviceSynchronize();
                    float ms; cudaEventElapsedTime(&ms, e0, e1);
                    printf("layout=%s ctas/sm=%d stages=%d hint=%s: %.1f us per 99.6 MB matrix = %.0f GB/s (%s)\n", tiled ? "tiled" : "rowmajor", per_sm,
                           stages, hintsel ? "evict_first" : "normal", ms * 1e3 / (reps * layers), per * 2.0 * reps * layers / (ms * 1e-3) / 1e9, cudaGetErrorString(err));
                }
    return 0;
}
