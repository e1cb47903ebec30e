// Codec input front end: PCM -> mono fp32, and the sinc resampler of torchaudio.functional.resample (defaults:
// sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99) on the device, for ragged batches of clips and for stream
// windows.
//
//   pcm_to_mono   interleaved int16 / int32 / uint8 / float32 frames -> mono fp32 with the arithmetic of the numpy
//                 reader (bulk_encode.read_audio): x / 32768, x / 2^31, (x - 128) / 128 in fp32, then the channels
//                 summed in order from 0.f and divided by the channel count (numpy's mean over a short axis).
//   resample      out[j] = sum_m w[m][p] * x(q * orig + first[p] + m), j = q * new + p, over the non-zero taps of
//                 phase p only, in ascending m, one fp64 fma each from 0.0, rounded to fp32 once. x(i) is 0 outside
//                 [0, x_end). The filter table is built on the host (fish_speech_b200/audio.py) in float64 and cast to
//                 fp32. The fp64 sum leaves the fp32 weights and the final rounding as the only errors: the result is
//                 closer to the float64 resample than torchaudio's fp32 one, whose table and sum are both fp32. The
//                 kernel moves 4 B in and 4 B out per output; the 13 - 27 fp64 fmas per output cost nothing beside it.
//   audio_out     the codec output front end: the same resampler from 44.1 kHz to the client's rate (or no resampling),
//                 each output rounded to fp32 once and stored as float32, or quantised in the same thread to int16
//                 PCM (utils.pcm16's rule) or 8-bit G.711 mu-law. 4 B in and 4, 2 or 1 B out per output.
// Each output depends on its own clip's samples and the table only, through one fixed sequence of operations: a clip
// gives the same bits alone or in any batch, and a stream window that holds every sample an output reads gives the
// same bits as the whole signal.
#include "../../include/fishb200.h"
#include "common.cuh"

using namespace fsb;

namespace {

constexpr int kAudioThreads = 256;

__device__ __forceinline__ float pcm_sample(const unsigned char* __restrict__ p, int fmt) {
    switch (fmt) {
        case FSB_PCM_S16: {
            const short v = static_cast<short>(p[0] | (p[1] << 8));
            return static_cast<float>(v) / 32768.0f;
        }
        case FSB_PCM_S32: {
            const int v = static_cast<int>(static_cast<unsigned>(p[0]) | (static_cast<unsigned>(p[1]) << 8) |
                                           (static_cast<unsigned>(p[2]) << 16) | (static_cast<unsigned>(p[3]) << 24));
            return static_cast<float>(v) / 2147483648.0f;
        }
        case FSB_PCM_U8:
            return (static_cast<float>(p[0]) - 128.0f) / 128.0f;
        default: {
            const unsigned u = static_cast<unsigned>(p[0]) | (static_cast<unsigned>(p[1]) << 8) |
                               (static_cast<unsigned>(p[2]) << 16) | (static_cast<unsigned>(p[3]) << 24);
            return __uint_as_float(u);
        }
    }
}

__device__ __forceinline__ int pcm_bytes(int fmt) { return fmt == FSB_PCM_S16 ? 2 : fmt == FSB_PCM_U8 ? 1 : 4; }

// One thread per frame of clip blockIdx.y. Byte loads: a clip's PCM may start at any byte offset of the buffer.
__global__ void __launch_bounds__(kAudioThreads)
pcm_to_mono_kernel(const unsigned char* __restrict__ src, const fsb_pcm_clip* __restrict__ clips,
                   float* __restrict__ dst) {
    pdl_launch_dependents();
    pdl_wait();
    const fsb_pcm_clip c = clips[blockIdx.y];
    const long long f = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (f >= c.frames) return;
    const int fmt = static_cast<int>(c.format), ch = static_cast<int>(c.channels), nb = pcm_bytes(fmt);
    const unsigned char* p = src + c.src_off + f * ch * nb;
    float acc = 0.f;
    for (int k = 0; k < ch; ++k) acc += pcm_sample(p + k * nb, fmt);
    dst[c.dst_off + f] = acc / static_cast<float>(ch);
}

// One thread per output j in [0, n_fill) of clip blockIdx.y: outputs j < n_out are absolute output j0 + j of the clip,
// the rest are zeros (the padding of a batch row).
__global__ void __launch_bounds__(kAudioThreads)
resample_kernel(const float* __restrict__ x, const fsb_resample_clip* __restrict__ clips, float* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const fsb_resample_clip c = clips[blockIdx.y];
    const long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j >= c.n_fill) return;
    double acc = 0.0;
    if (j < c.n_out) {
        const long long a = c.j0 + j;
        const float* xs = x + c.x_off - c.x_start;  // xs[i] = sample i, for x_start <= i < x_end
        if (c.w == nullptr) {
            acc = (a >= 0 && a < c.x_end) ? xs[a] : 0.f;
        } else {
            const long long q = a / c.new_rate;
            const int p = static_cast<int>(a - q * c.new_rate);
            const int2 span = reinterpret_cast<const int2*>(c.span)[p];  // (first tap offset, non-zero taps)
            const long long i0 = q * c.orig + span.x;
            for (int m = 0; m < span.y; ++m) {
                const long long i = i0 + m;
                const float v = (i >= 0 && i < c.x_end) ? __ldg(xs + i) : 0.f;
                acc = fma(static_cast<double>(__ldg(c.w + static_cast<long long>(m) * c.new_rate + p)),
                          static_cast<double>(v), acc);
            }
        }
    }
    out[c.out_off + j] = static_cast<float>(acc);
}

// resample_kernel's arithmetic for absolute output a of an output row: the same taps in the same order, one fp64 fma
// each from 0.0 (kept apart from resample_kernel so that kernel's code stays as it was built).
__device__ __forceinline__ double resample_at(const float* __restrict__ x, const fsb_audio_out_row& c, long long a) {
    const float* xs = x + c.x_off - c.x_start;  // xs[i] = sample i, for x_start <= i < x_end
    if (c.w == nullptr) return (a >= 0 && a < c.x_end) ? xs[a] : 0.f;
    double acc = 0.0;
    const long long q = a / c.new_rate;
    const int p = static_cast<int>(a - q * c.new_rate);
    const int2 span = reinterpret_cast<const int2*>(c.span)[p];
    const long long i0 = q * c.orig + span.x;
    for (int m = 0; m < span.y; ++m) {
        const long long i = i0 + m;
        const float v = (i >= 0 && i < c.x_end) ? __ldg(xs + i) : 0.f;
        acc = fma(static_cast<double>(__ldg(c.w + static_cast<long long>(m) * c.new_rate + p)),
                  static_cast<double>(v), acc);
    }
    return acc;
}

// utils.pcm16 of one fp32 sample: trunc(min(max(y, -1), 1) * 32767.0f), the multiply rounded to nearest on its own
// (no fma contraction), the conversion truncating toward zero. The comparisons keep a NaN, which converts to 0.
__device__ __forceinline__ int pcm16_of(float y) {
    y = y < -1.f ? -1.f : (y > 1.f ? 1.f : y);
    return __float2int_rz(__fmul_rn(y, 32767.0f));
}

// G.711 mu-law of a 16-bit sample (the Sun g711.c encoder that audioop.lin2ulaw runs): the sample shifted to 14 bits,
// its magnitude clipped to 8159 and biased by 33 (132 >> 2), segment = position of its top bit above bit 5, four
// mantissa bits below it, every bit inverted (the sign bit only for non-negative samples).
__device__ __forceinline__ unsigned char mulaw_of(int s) {
    int v = s >> 2;  // arithmetic: floor(s / 4)
    int mask = 0xFF;
    if (v < 0) {
        v = -v;
        mask = 0x7F;
    }
    v = min(v, 8159) + 33;
    int seg = 0;
    while (seg < 8 && v > (0x40 << seg) - 1) ++seg;
    if (seg >= 8) return static_cast<unsigned char>(0x7F ^ mask);
    return static_cast<unsigned char>(((seg << 4) | ((v >> (seg + 1)) & 0xF)) ^ mask);
}

// One thread per output j in [0, n_out) of row blockIdx.y: absolute output j0 + j, rounded to fp32 once as
// resample_kernel rounds it, then stored in the row's format at byte offset out_off + j * (4, 2 or 1).
__global__ void __launch_bounds__(kAudioThreads)
audio_out_kernel(const float* __restrict__ x, const fsb_audio_out_row* __restrict__ rows, unsigned char* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const fsb_audio_out_row c = rows[blockIdx.y];
    const long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j >= c.n_out) return;
    const float y = static_cast<float>(resample_at(x, c, c.j0 + j));
    unsigned char* o = out + c.out_off;
    switch (static_cast<int>(c.format)) {
        case FSB_OUT_F32:
            reinterpret_cast<float*>(o)[j] = y;
            break;
        case FSB_OUT_PCM16:
            reinterpret_cast<short*>(o)[j] = static_cast<short>(pcm16_of(y));
            break;
        default:
            o[j] = mulaw_of(pcm16_of(y));
            break;
    }
}

}  // namespace

int fsb_pcm_to_mono(const void* d_src, const fsb_pcm_clip* d_clips, int B, long long max_frames, float* d_dst,
                    void* stream) {
    FSB_CHECK(B >= 0 && B <= 65535 && max_frames >= 0, "pcm_to_mono: B=%d max_frames=%lld", B, max_frames);
    if (B == 0 || max_frames == 0) return 0;
    FSB_CHECK(cdivll(max_frames, kAudioThreads) <= 0x7fffffffll, "pcm_to_mono: %lld frames", max_frames);
    FSB_LAUNCH(pcm_to_mono_kernel, dim3(static_cast<unsigned>(cdivll(max_frames, kAudioThreads)), B),
               dim3(kAudioThreads), 0, reinterpret_cast<cudaStream_t>(stream),
               reinterpret_cast<const unsigned char*>(d_src), d_clips, d_dst);
    return 0;
}

int fsb_resample(const float* d_x, const fsb_resample_clip* d_clips, int B, long long max_fill, float* d_out,
                 void* stream) {
    FSB_CHECK(B >= 0 && B <= 65535 && max_fill >= 0, "resample: B=%d max_fill=%lld", B, max_fill);
    if (B == 0 || max_fill == 0) return 0;
    FSB_CHECK(cdivll(max_fill, kAudioThreads) <= 0x7fffffffll, "resample: %lld outputs", max_fill);
    FSB_LAUNCH(resample_kernel, dim3(static_cast<unsigned>(cdivll(max_fill, kAudioThreads)), B), dim3(kAudioThreads),
               0, reinterpret_cast<cudaStream_t>(stream), d_x, d_clips, d_out);
    return 0;
}

int fsb_audio_out(const float* d_x, const fsb_audio_out_row* d_rows, int B, long long max_out, void* d_out,
                  void* stream) {
    FSB_CHECK(B >= 0 && B <= 65535 && max_out >= 0, "audio_out: B=%d max_out=%lld", B, max_out);
    if (B == 0 || max_out == 0) return 0;
    FSB_CHECK(cdivll(max_out, kAudioThreads) <= 0x7fffffffll, "audio_out: %lld outputs", max_out);
    FSB_LAUNCH(audio_out_kernel, dim3(static_cast<unsigned>(cdivll(max_out, kAudioThreads)), B), dim3(kAudioThreads),
               0, reinterpret_cast<cudaStream_t>(stream), d_x, d_rows, reinterpret_cast<unsigned char*>(d_out));
    return 0;
}
