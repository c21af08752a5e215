// Downmix + polyphase resampling of any-rate, any-channel waveforms to the 16 kHz mono the frontend is built for
// (whisper_b200.h wb_resample): scipy.signal.resample_poly(x, up, down) with its default Kaiser (beta 5) FIR, in f64.
//   x[i]  = (x[i,0] + .. + x[i,C-1]) / C                                   f64, channel order
//   y[k]  = sum_i h[half + k*down - i*up] * x[i]   over 0 <= half + k*down - i*up <= 2*half, 0 <= i < n
//   h[j]  = up * w[j] / sum(w),  w[j] = sinc((j - half) / m) * kaiser(2*half + 1, 5.0)[j],  m = max(up, down), half = 10*m
// y[k] is rounded once to f32; up = down = 1 is h = [1], so 16 kHz mono passes through bit-unchanged.
#include <cmath>
#include <numeric>

#include "wb_internal.h"

namespace wb {

constexpr int RS_THREADS = 256;   // one output per thread: a tile is RS_THREADS consecutive outputs of one waveform
constexpr int RS_SPAN = 4096;     // downmixed input frames staged per pass (32 KB of f64); longer spans take several passes

// Output tiles of all waveforms of the call are dealt over the grid (desc[w].tile0: the first tile of waveform w), so a short
// waveform occupies as many CTAs as it has tiles.  Each CTA stages the input frames its tile reads, downmixed once per frame,
// then every output walks only the taps that land on input samples: j = half + k*down - i*up steps down by `up`.
// Outside the anonymous namespace so that profiles find it by a stable name.
__global__ void __launch_bounds__(RS_THREADS)
resample_poly_kernel(const float* __restrict__ in, const ResampleDesc* __restrict__ desc, int n_desc,
                     const double* __restrict__ taps, float* __restrict__ out, int64_t n_tiles) {
    __shared__ double xs[RS_SPAN];
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        int lo = 0, hi = n_desc - 1;   // the waveform of this tile: the last descriptor with tile0 <= tile
        while (lo < hi) {
            const int mid = (lo + hi + 1) / 2;
            if (desc[mid].tile0 <= tile) lo = mid;
            else hi = mid - 1;
        }
        const ResampleDesc d = desc[lo];
        const int64_t k0 = (tile - d.tile0) * RS_THREADS;
        const int64_t k1 = min(k0 + RS_THREADS, d.n_out);
        const int64_t k = k0 + threadIdx.x;
        const bool live = k < k1;
        // the input frames output k reads: ceil((k*down - half) / up) .. floor((k*down + half) / up), clipped to the input
        auto first_frame = [&](int64_t kk) {
            const int64_t t = kk * d.down - d.half;
            return t <= 0 ? (int64_t)0 : (t + d.up - 1) / d.up;
        };
        auto last_frame = [&](int64_t kk) { return min((kk * d.down + d.half) / d.up, d.n - 1); };
        const int64_t span_lo = first_frame(k0), span_hi = last_frame(k1 - 1);
        const int64_t my_lo = live ? first_frame(k) : 0, my_hi = live ? last_frame(k) : -1;
        const float* x = in + d.in_off;
        const double* h = taps + d.taps_off;
        const double n_ch = (double)d.channels;
        double acc = 0.0;
        for (int64_t c0 = span_lo; c0 <= span_hi; c0 += RS_SPAN) {
            const int64_t c1 = min(c0 + RS_SPAN - 1, span_hi);
            __syncthreads();   // every thread is done with the previous pass (or tile)
            for (int64_t f = c0 + threadIdx.x; f <= c1; f += RS_THREADS) {
                const float* p = x + f * d.channels;
                double s = 0.0;
                for (int c = 0; c < d.channels; ++c) s += (double)__ldg(p + c);
                xs[f - c0] = s / n_ch;
            }
            __syncthreads();
            const int64_t ia = max(my_lo, c0), ib = min(my_hi, c1);
            int64_t j = d.half + k * d.down - ia * d.up;
            for (int64_t i = ia; i <= ib; ++i, j -= d.up) acc = fma(__ldg(h + j), xs[i - c0], acc);
        }
        if (live) out[d.out_off + k] = (float)acc;
    }
}

namespace {

// modified Bessel function of the first kind, order 0 (numpy.i0), by its power series: sum ((x/2)^k / k!)^2
double bessel_i0(double x) {
    double sum = 1.0, term = 1.0;
    const double q = 0.25 * x * x;
    for (int k = 1; k < 500; ++k) {
        term *= q / ((double)k * k);
        sum += term;
        if (term < 1e-17 * sum) break;
    }
    return sum;
}

}  // namespace

bool resample_ratio(int64_t sample_rate, int& up, int& down) {
    if (sample_rate < 1) return false;
    const int64_t g = std::gcd(sample_rate, (int64_t)16000);
    if (16000 / g > 1024 || sample_rate / g > 1024) return false;
    up = (int)(16000 / g);
    down = (int)(sample_rate / g);
    return true;
}

int64_t resampled_length(int64_t n_frames, int64_t sample_rate) {
    int up = 0, down = 0;
    if (n_frames < 0 || !resample_ratio(sample_rate, up, down)) return -1;
    if (n_frames > (INT64_MAX - down) / up) return -1;
    return (n_frames * up + down - 1) / down;   // ceil(n * up / down)
}

std::vector<double> resample_taps(int up, int down) {
    if (up == 1 && down == 1) return {1.0};   // resample_poly's copy
    const int m = std::max(up, down), half = 10 * m, N = 2 * half + 1;
    const double beta = 5.0, i0_beta = bessel_i0(beta), pi = 3.14159265358979323846;
    std::vector<double> h((size_t)N);
    double sum = 0.0;
    for (int j = 0; j < N; ++j) {
        const double t = (double)(j - half) / m;
        const double sinc = t == 0.0 ? 1.0 : std::sin(pi * t) / (pi * t);
        const double r = (double)(j - half) / half;
        h[(size_t)j] = sinc * bessel_i0(beta * std::sqrt(std::max(0.0, 1.0 - r * r))) / i0_beta;
        sum += h[(size_t)j];
    }
    for (double& v : h) v = up * v / sum;
    return h;
}

void resample_waveforms(ResampleBufs& b, const float* const* in, const int64_t* n_frames, const int64_t* channels,
                        const int64_t* sample_rates, int64_t n_waveforms, std::vector<int64_t>& out_off,
                        std::vector<int64_t>& n_out, cudaStream_t st) {
    std::vector<ResampleDesc> desc((size_t)n_waveforms);
    std::vector<double> taps;
    std::vector<std::pair<int64_t, int64_t>> designed;   // (rate, offset into taps): one filter per distinct rate of the call
    out_off.assign((size_t)n_waveforms, 0);
    n_out.assign((size_t)n_waveforms, 0);
    int64_t in_total = 0, out_total = 0, tiles = 0;
    for (int64_t w = 0; w < n_waveforms; ++w) {
        ResampleDesc& d = desc[(size_t)w];
        int up = 0, down = 0;
        if (!resample_ratio(sample_rates[w], up, down)) fail(WB_ERR_UNSUPPORTED, "resample: unsupported sample rate");
        d.in_off = in_total;
        d.n = n_frames[w];
        d.channels = (int)channels[w];
        d.up = up;
        d.down = down;
        d.half = up == 1 && down == 1 ? 0 : 10 * std::max(up, down);
        d.out_off = out_total;
        d.n_out = resampled_length(n_frames[w], sample_rates[w]);
        d.tile0 = tiles;
        auto it = std::find_if(designed.begin(), designed.end(), [&](const auto& p) { return p.first == sample_rates[w]; });
        if (it == designed.end()) {
            designed.emplace_back(sample_rates[w], (int64_t)taps.size());
            const std::vector<double> h = resample_taps(up, down);
            taps.insert(taps.end(), h.begin(), h.end());
            it = designed.end() - 1;
        }
        d.taps_off = it->second;
        out_off[(size_t)w] = out_total;
        n_out[(size_t)w] = d.n_out;
        in_total += d.n * d.channels;
        out_total += d.n_out;
        tiles += (d.n_out + RS_THREADS - 1) / RS_THREADS;
    }
    b.in.ensure((size_t)in_total);
    b.out.ensure((size_t)std::max<int64_t>(out_total, 1));
    b.taps.ensure(taps.size());
    b.desc.ensure(desc.size());
    for (int64_t w = 0; w < n_waveforms; ++w)
        WB_CUDA(cudaMemcpyAsync(b.in.p + desc[(size_t)w].in_off, in[w], (size_t)(desc[(size_t)w].n * desc[(size_t)w].channels) * sizeof(float),
                                cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(b.taps.p, taps.data(), taps.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    WB_CUDA(cudaMemcpyAsync(b.desc.p, desc.data(), desc.size() * sizeof(ResampleDesc), cudaMemcpyHostToDevice, st));
    if (tiles > 0) {
        resample_poly_kernel<<<(unsigned)std::min<int64_t>(tiles, 65535), RS_THREADS, 0, st>>>(b.in.p, b.desc.p, (int)n_waveforms,
                                                                                              b.taps.p, b.out.p, tiles);
        WB_LAUNCH_CHECK();
    }
    WB_CUDA(cudaStreamSynchronize(st));   // the host descriptors and filters above are temporaries
}

}  // namespace wb
