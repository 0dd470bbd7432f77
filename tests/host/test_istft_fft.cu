// Host-side check of the inverse-FFT lane code (flowtron_b200/csrc/mel_fft.cuh: inv_pretwiddle, the forward passes,
// inv_readout) as istft.cu runs it, for all 32 "lanes" sequentially, against a direct O(N^2) double-precision inverse
// real DFT.  The spectra have non-zero imaginary parts at DC and Nyquist, which an irfft ignores.
// Build + run: nvcc -std=c++17 -I flowtron_b200/csrc tests/host/test_istft_fft.cu -o test_istft_fft && ./test_istft_fft
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "mel_fft.cuh"

using namespace ft::melfft;

struct Src {
    const cf* X;
    const float2* tw;
    float2 operator()(int n) const {
        const cf z = inv_pretwiddle(n, X[n], X[NH - n], tw);
        return make_float2(z.x, z.y);
    }
};

int main() {
    std::vector<float2> tw(1024);
    for (int j = 0; j < 1024; ++j) { const double a = -2.0 * M_PI * j / 1024.0; tw[j] = make_float2((float)cos(a), (float)sin(a)); }
    double worst = 0.0;
    for (int trial = 0; trial < 6; ++trial) {
        std::vector<cf> X(NBINS);
        srand(29 + trial);
        for (auto& v : X) {
            const float m = trial >= 3 ? (float)rand() / RAND_MAX : 1.0f, ph = ((float)rand() / RAND_MAX * 2.f - 1.f) * 3.14159265f;
            v = {m * cosf(ph), m * sinf(ph)};
        }
        std::vector<float> xr(XBUF), xi(XBUF);
        Src src{X.data(), tw.data()};
        for (int lane = 0; lane < 32; ++lane) for (int h = 0; h < 2; ++h) pass_a(lane + 32 * h, src, tw.data(), xr.data(), xi.data());
        cf regs[32][2][8];
        for (int lane = 0; lane < 32; ++lane) for (int h = 0; h < 2; ++h) pass_b_load(lane + 32 * h, xr.data(), xi.data(), regs[lane][h]);
        for (int lane = 0; lane < 32; ++lane) for (int h = 0; h < 2; ++h) pass_b_store(lane + 32 * h, regs[lane][h], tw.data(), xr.data(), xi.data());
        for (int lane = 0; lane < 32; ++lane) for (int h = 0; h < 2; ++h) pass_c_load(lane + 32 * h, xr.data(), xi.data(), regs[lane][h]);
        for (int lane = 0; lane < 32; ++lane) for (int h = 0; h < 2; ++h) pass_c_store(lane + 32 * h, regs[lane][h], xr.data(), xi.data());
        // x[n] = (1/N) (Re X0 + Re X512 (-1)^n + 2 sum_{k=1}^{511} Re(X[k] e^{2 pi i k n / N}))
        std::vector<double> ref(NFFT);
        double scale = 0.0;
        for (int n = 0; n < NFFT; ++n) {
            double s = X[0].x + ((n & 1) ? -X[NH].x : X[NH].x);
            for (int k = 1; k < NH; ++k) {
                const double a = 2.0 * M_PI * (double)k * n / NFFT;
                s += 2.0 * (X[k].x * cos(a) - X[k].y * sin(a));
            }
            ref[n] = s / NFFT;
            scale = fmax(scale, fabs(ref[n]));
        }
        for (int n = 0; n < NFFT; ++n) worst = fmax(worst, fabs(inv_readout(n, xr.data(), xi.data()) - ref[n]) / scale);
    }
    printf("istft_fft host check: worst relative error %.3e\n", worst);
    return worst <= 1e-6 ? 0 : 1;
}
