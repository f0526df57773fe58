// Host-logic check of cpp/phastft.hpp (CPU-only part runs without a GPU; with a GPU it also runs the
// reference's doctest lib.rs:171-178).  Built and run by tests/test_cpu_cpp_mirror.py.
#include <cmath>
#include <cstdio>
#include <cstring>
#include "phastft.hpp"

template <typename F>
static bool panics_with(F f, const char* msg) {
    try { f(); } catch (const phastft::Panic& e) { return std::strstr(e.what(), msg) != nullptr; }
    return false;
}

int main() {
    using namespace phastft;
    int fails = 0;
    // planner.rs:66 / planner.rs:195 are checked before any device is touched
    fails += !panics_with([] { PlannerDit64 p(5); }, "power of two");
    fails += !panics_with([] { PlannerDit32 p(0); }, "power of two");
    fails += !panics_with([] { PlannerR2c64 p(6); }, "n must be a power of 2 >= 4");
    fails += !panics_with([] { PlannerDct64 p(0); }, "n must be >= 1");
    fails += !panics_with([] { PlannerConv64 p(0, 5); }, "n_x and n_h must be >= 1");
    fails += !panics_with([] { PlannerStft64 p(32, 64, 16); }, "reflect padding");
    fails += !panics_with([] { PlannerStft32 p(100, 64, 0); }, "hop must be >= 1");
    fails += !panics_with([] { PlannerConv32 p(std::size_t(1) << 30, 2, 0, true); }, "above 2^30");
    fails += conv_out_len(10, 4, ConvMode::Full) != 13 || conv_out_len(10, 4, ConvMode::Same) != 10 || conv_out_len(4, 10, ConvMode::Valid) != 7;
    fails += !panics_with([] { std::vector<float> x(2), a(2), b(2); r2c_fft_f32(x, a, b); }, "n must be a power of 2 >= 4");
    Options o = Options::guess_options(1 << 16);
    fails += !(o.multithreaded_bit_reversal && o.smallest_parallel_chunk_size == 16384);
    int ndev = 0;
    phastft_device_count(&ndev);
    if (ndev == 0) {
        fails += !panics_with([] { PlannerDit64 p(1024); }, "no CUDA device");
        std::printf("cpu-only checks: %d failures\n", fails);
        return fails;
    }
    std::vector<double> re{1, 0, 0, 0}, im(4, 0.0);
    fft_64_dit(re, im, Direction::Forward);
    for (double v : re) fails += std::fabs(v - 1.0) > 1e-12;
    fails += !panics_with([] { std::vector<double> a(16), b(8); PlannerDit64 p(16); fft_64_dit_with_planner(a, b, Direction::Forward, p); }, "reals.len() == imags.len()");
    {   // additive surface: describe / reserve / batch == loop over transforms (bit-exact below the batched-kernel threshold)
        const std::size_t n = 256, batch = 5, stride = n + 8;
        PlannerDit32 p(n);
        fails += p.num_points() != n || p.describe().find("n=2^8") == std::string::npos;
        p.reserve(batch);
        std::vector<float> bre(batch * stride), bim(batch * stride);
        for (std::size_t i = 0; i < bre.size(); ++i) { bre[i] = std::sin(0.37f * i); bim[i] = std::cos(0.11f * i); }
        std::vector<float> lre = bre, lim = bim;
        fft_32_dit_batch(bre, bim, Direction::Forward, p, batch, stride);
        for (std::size_t b = 0; b < batch; ++b) {
            std::vector<float> a(lre.begin() + b * stride, lre.begin() + b * stride + n), c(lim.begin() + b * stride, lim.begin() + b * stride + n);
            fft_32_dit_with_planner(a, c, Direction::Forward, p);
            for (std::size_t i = 0; i < n; ++i) fails += a[i] != bre[b * stride + i] || c[i] != bim[b * stride + i];
        }
    }
    {   // additive surface: DCT-II then DCT-III of it, divided by 2N, gives the input back; in place on the host
        const std::size_t n = 1000;
        PlannerDct64 p(n);
        fails += p.n() != n || p.describe().find("n=1000 f64 dct | ") != 0;
        std::vector<double> x(n), y(n);
        for (std::size_t i = 0; i < n; ++i) x[i] = std::sin(0.37 * i);
        p.transform(R2rKind::Dct2, R2rNorm::Backward, x, y);
        p.transform(R2rKind::Dct3, R2rNorm::Forward, y, y);
        for (std::size_t i = 0; i < n; ++i) fails += std::fabs(y[i] - x[i]) > 1e-12;
    }
    {   // additive surface: convolution and correlation against direct sums, real and complex
        const std::size_t nx = 300, nh = 37;
        PlannerConv64 p(nx, nh);
        fails += p.fft_len() != 512 || p.describe().find("n_x=300 n_h=37 f64 conv real L=2^9 | ") != 0;
        std::vector<double> x(nx), h(nh), y(p.out_len(ConvMode::Valid));
        for (std::size_t i = 0; i < nx; ++i) x[i] = std::sin(0.37 * i);
        for (std::size_t i = 0; i < nh; ++i) h[i] = std::cos(0.21 * i);
        p.convolve(x, h, y, ConvMode::Valid);
        for (std::size_t j = 0; j < y.size(); ++j) {
            double s = 0;
            for (std::size_t k = 0; k < nh; ++k) s += x[j + nh - 1 - k] * h[k];
            fails += std::fabs(y[j] - s) > 1e-12;
        }
        fails += !panics_with([&] { std::vector<std::complex<double>> a(nx), b(nh), c(nx); p.convolve(a, b, c, ConvMode::Same); }, "domain mismatch");
        PlannerConv32 q(nx, nh, 0, true);
        fails += !panics_with([&] { std::vector<float> a(nx), b(nh), c(nx + nh - 1); q.correlate(a, b, c); }, "domain mismatch");
        std::vector<std::complex<float>> cx(nx), ch(nh), cy(q.out_len(ConvMode::Valid));
        for (std::size_t i = 0; i < nx; ++i) cx[i] = {std::sin(0.37f * i), std::cos(0.5f * i)};
        for (std::size_t i = 0; i < nh; ++i) ch[i] = {std::cos(0.21f * i), 0.25f};
        q.correlate(cx, ch, cy, ConvMode::Valid);
        for (std::size_t j = 0; j < cy.size(); ++j) {
            std::complex<double> s = 0;
            for (std::size_t k = 0; k < nh; ++k) s += std::complex<double>(cx[j + k]) * std::conj(std::complex<double>(ch[k]));
            fails += std::abs(std::complex<double>(cy[j]) - s) > 1e-4;
        }
    }
    {   // additive surface: a round trip through the STFT, real and complex
        const std::size_t n = 4000, nf = 400, hop = 100;
        std::vector<double> w(nf);
        for (std::size_t i = 0; i < nf; ++i) w[i] = 0.5 - 0.5 * std::cos(2 * 3.14159265358979323846 * i / nf);
        PlannerStft64 p(n, nf, hop, w);
        fails += p.frames() != 41 || p.bins() != 201 || p.describe().find("n=4000 n_fft=400 hop=100 f64 stft real F=41 | ") != 0;
        std::vector<double> x(n), y(n);
        for (std::size_t i = 0; i < n; ++i) x[i] = std::sin(0.37 * i);
        std::vector<std::complex<double>> spec(p.frames() * p.bins());
        p.stft(x, spec);
        p.istft(spec, y);
        for (std::size_t i = 0; i < n; ++i) fails += std::fabs(y[i] - x[i]) > 1e-12;
        fails += !panics_with([&] { std::vector<std::complex<double>> c(n); p.stft(c, spec); }, "domain mismatch");
        PlannerStft32 q(n, 512, 128, {}, 0, false, StftPad::Constant, 0, true);
        std::vector<std::complex<float>> cx(n), cy(n), cs(q.frames() * q.bins());
        for (std::size_t i = 0; i < n; ++i) cx[i] = {std::sin(0.37f * i), std::cos(0.5f * i)};
        q.stft(cx, cs);
        q.istft(cs, cy);
        const std::size_t covered = 512 + 128 * (q.frames() - 1);
        for (std::size_t i = 0; i < covered; ++i) fails += std::abs(cy[i] - cx[i]) > 1e-5f;
    }
    std::printf("gpu checks: %d failures\n", fails);
    return fails;
}
