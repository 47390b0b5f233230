// sonicsim_b200 :: ss_dry.cu - dry-stream assembly on the device (SURVEY 8f rank 2).
//
// The arithmetic of SonicSim_audio.create_long_audio / create_background_audio (SonicSim_audio.py:231-340) once
// the host has drawn which clip goes where: per placed clip
//   1. torchaudio.transforms.Resample(orig, new) (:253-256, :300-303) - the polyphase sinc / Hann filter bank
//      y[j * new + p] = sum_k K[p][k] * xpad[j * orig + k],  xpad = x padded by `width` zeros on the left
//      (torchaudio.functional._apply_sinc_resample_kernel), per channel;
//   2. stereo -> mono `audio.mean(dim=0)` (:311-312): (a + b) / 2 after the resampling, as the reference orders it;
//   3. `long_audio[:, a:b] += clip[...]` onto the zero-initialised stream (:268, :326, :332).
// One kernel over (clip, output tile); the stream never leaves HBM, so it can feed ss_render_dev / ss_plan_run
// directly.  fp32 accumulation in tap order; the reference's conv1d (oneDNN) sums in another order, so resampled
// clips agree to rounding (~1e-7 relative), un-resampled ones bit for bit.
#include <string.h>

#include <algorithm>
#include <utility>

#include "ss_internal.h"

namespace {

struct DryClip {
    const float* src;        // (channels, src_len)
    const float* kernel_t;   // (taps, new_) transposed filter bank, or null: no resampling
    long long dst_start, src_start, count;
    int channels, src_len, orig, new_, width, taps;
};

__device__ __forceinline__ float resampled_at(const DryClip& c, const float* x, long long m) {
    if (!c.kernel_t) return x[m];
    const long long j = m / c.new_;
    const int p = (int)(m - j * c.new_);
    const long long base = j * c.orig - c.width;          // xpad[i] = x[i - width]
    const float* kp = c.kernel_t + p;
    int k0 = base < 0 ? (int)(-base) : 0;
    int k1 = c.taps;
    if (base + k1 > c.src_len) k1 = (int)(c.src_len - base);
    float acc = 0.f;
    for (int k = k0; k < k1; ++k) acc = fmaf(kp[(size_t)k * c.new_], x[base + k], acc);
    return acc;
}

__global__ void __launch_bounds__(256) k_dry_assemble(const DryClip* __restrict__ clips, float* __restrict__ out) {
    const DryClip& c = clips[blockIdx.y];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < c.count; i += (long long)gridDim.x * blockDim.x) {
        const long long m = c.src_start + i;
        float v = resampled_at(c, c.src, m);
        if (c.channels == 2) {
            const float b = resampled_at(c, c.src + c.src_len, m);
            v = __fmul_rn(__fadd_rn(v, b), 0.5f);          // torch.mean over 2 channels: (a + b) / 2
        }
        out[c.dst_start + i] += v;                         // += onto the zeroed stream, as the reference writes it
    }
}

}  // namespace

extern "C" int ss_dry_assemble_dev(ss_ctx* c, const ss_dry_clip* clips, int n_clips, float* out, int64_t total, void* stream_) {
    if (!c || !out || total <= 0 || n_clips < 0 || (n_clips > 0 && !clips)) return SS_ERR_INVALID;
    if (n_clips > 65535) return SS_ERR_UNSUPPORTED;             // one gridDim.y row per clip
    cudaStream_t stream = (cudaStream_t)stream_;
    std::vector<std::pair<int64_t, int64_t>> ranges;            // destination [start, end) of every non-empty clip
    for (int i = 0; i < n_clips; ++i) {
        const ss_dry_clip& k = clips[i];
        if (!k.src || k.channels < 1 || k.channels > 2 || k.src_len <= 0 || k.count < 0) return SS_ERR_INVALID;
        if (k.dst_start < 0 || k.src_start < 0 || k.dst_start + k.count > total) return SS_ERR_INVALID;
        if (k.kernel_t) {
            if (k.orig <= 0 || k.new_rate <= 0 || k.width < 0 || k.taps != 2 * k.width + k.orig) return SS_ERR_INVALID;
            const int64_t res_len = ((int64_t)k.new_rate * k.src_len + k.orig - 1) / k.orig;      // ceil(new * len / orig)
            if (k.src_start + k.count > res_len) return SS_ERR_INVALID;
        } else if (k.src_start + k.count > k.src_len) return SS_ERR_INVALID;
        if (k.count > 0) ranges.emplace_back(k.dst_start, k.dst_start + k.count);
    }
    // clips add onto the stream from different CTAs without atomics, so no two may write the same sample
    std::sort(ranges.begin(), ranges.end());
    for (size_t i = 1; i < ranges.size(); ++i)
        if (ranges[i].first < ranges[i - 1].second) return SS_ERR_INVALID;
    CK(cudaSetDevice(c->device));
    CK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)total, stream));
    if (n_clips == 0) return SS_OK;
    const size_t bytes = sizeof(DryClip) * (size_t)n_clips;
    int slot; char *hblk, *dblk;
    { int st = ring_acquire(c, bytes, stream, &slot, &hblk, &dblk); if (st) return st; }
    DryClip* h = (DryClip*)hblk;
    long long max_count = 1;
    for (int i = 0; i < n_clips; ++i) {
        const ss_dry_clip& k = clips[i];
        DryClip d; memset(&d, 0, sizeof(d));
        d.src = k.src; d.kernel_t = k.kernel_t; d.dst_start = k.dst_start; d.src_start = k.src_start; d.count = k.count;
        d.channels = k.channels; d.src_len = k.src_len; d.orig = k.orig; d.new_ = k.new_rate; d.width = k.width; d.taps = k.taps;
        h[i] = d;
        if (k.count > max_count) max_count = k.count;
    }
    CK(cudaMemcpyAsync(dblk, hblk, bytes, cudaMemcpyHostToDevice, stream));
    CK(cudaEventRecord(c->desc_ev[slot], stream));
    const unsigned gx = (unsigned)((max_count + 255) / 256 < 2048 ? (max_count + 255) / 256 : 2048);
    k_dry_assemble<<<dim3(gx, (unsigned)n_clips), 256, 0, stream>>>((const DryClip*)dblk, out);
    CK(cudaGetLastError());
    c->launches += 1;
    return ring_release(c, slot, stream);
}
