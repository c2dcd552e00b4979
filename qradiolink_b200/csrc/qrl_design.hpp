// qrl_design.hpp -- host-side filter / table / loop-gain design for the GPU path.
//
// These are the construction-time computations the reference performs through GNU Radio's
// gr::filter::firdes, gr::fft::window, gr::calculate_deemph_taps and the control-loop constructors
// (call sites: /root/reference/src/gr/gr_demod_4fsk.cpp:98-128, gr_demod_qpsk.cpp:98-120,
// gr_demod_nbfm.cpp:44-66, gr_mod_4fsk.cpp:78-92, emphasis.cpp:16-88).  They run once per handle on
// the host in double precision and the results are uploaded to HBM; nothing here is on the hot path.
#pragma once
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

namespace qrl {

enum Window { WIN_HAMMING = 0, WIN_HANN = 1, WIN_BLACKMAN = 2, WIN_RECT = 3, WIN_KAISER = 4, WIN_BLACKMAN_HARRIS = 5 };

static const double kPi = 3.14159265358979323846;

inline double window_max_attenuation(int win)
{
    switch (win) {
    case WIN_HAMMING: return 53; case WIN_HANN: return 44; case WIN_BLACKMAN: return 74;
    case WIN_RECT: return 21; case WIN_BLACKMAN_HARRIS: return 92; default: return 53;
    }
}

// gr::fft::window::build (cosine-sum windows are evaluated with cosf on a float argument)
inline std::vector<float> window_build(int win, int ntaps)
{
    std::vector<float> w(ntaps);
    const float M = static_cast<float>(ntaps - 1);
    for (int n = 0; n < ntaps; n++) {
        if (win == WIN_HAMMING) w[n] = static_cast<float>(0.54 - 0.46 * std::cos((2 * kPi * n) / M));
        else if (win == WIN_HANN) w[n] = static_cast<float>(0.5 - 0.5 * std::cos((2 * kPi * n) / M));
        else if (win == WIN_BLACKMAN) {
            const float c0 = 0.42f, c1 = 0.5f, c2 = 0.08f;
            w[n] = c0 - c1 * cosf(static_cast<float>((2.0 * kPi * n) / M)) + c2 * cosf(static_cast<float>((4.0 * kPi * n) / M));
        } else if (win == WIN_BLACKMAN_HARRIS) {
            const float c0 = 0.35875f, c1 = 0.48829f, c2 = 0.14128f, c3 = 0.01168f;
            w[n] = c0 - c1 * cosf(static_cast<float>((2.0 * kPi * n) / M)) + c2 * cosf(static_cast<float>((4.0 * kPi * n) / M))
                   - c3 * cosf(static_cast<float>((6.0 * kPi * n) / M));
        } else w[n] = 1.0f;
    }
    return w;
}

inline int ntaps_for_window(double fs, double tw, int win)
{
    int n = static_cast<int>(window_max_attenuation(win) * fs / (22.0 * tw));
    return (n & 1) ? n : n + 1;
}
inline int ntaps_for_attenuation(double fs, double tw, double att_db)
{
    int n = static_cast<int>(att_db * fs / (22.0 * tw));
    return (n & 1) ? n : n + 1;
}

inline std::vector<float> low_pass_core(double gain, double fs, double fc, int ntaps, int win)
{
    std::vector<float> taps(ntaps), w = window_build(win, ntaps);
    const int M = (ntaps - 1) / 2;
    const double wc = 2 * kPi * fc / fs;
    for (int n = -M; n <= M; n++)
        taps[n + M] = (n == 0) ? static_cast<float>(wc / kPi * w[n + M]) : static_cast<float>(std::sin(n * wc) / (n * kPi) * w[n + M]);
    double dc = taps[M];
    for (int n = 1; n <= M; n++) dc += 2 * taps[n + M];
    gain /= dc;
    for (auto& t : taps) t = static_cast<float>(t * gain);
    return taps;
}
inline std::vector<float> low_pass(double gain, double fs, double fc, double tw, int win = WIN_HAMMING)
{ return low_pass_core(gain, fs, fc, ntaps_for_window(fs, tw, win), win); }
inline std::vector<float> low_pass_2(double gain, double fs, double fc, double tw, double att_db, int win = WIN_HAMMING)
{ return low_pass_core(gain, fs, fc, ntaps_for_attenuation(fs, tw, att_db), win); }

inline std::vector<float> band_pass_core(double gain, double fs, double lo, double hi, int ntaps, int win)
{
    std::vector<float> taps(ntaps), w = window_build(win, ntaps);
    const int M = (ntaps - 1) / 2;
    const double w0 = 2 * kPi * lo / fs, w1 = 2 * kPi * hi / fs;
    for (int n = -M; n <= M; n++)
        taps[n + M] = (n == 0) ? static_cast<float>((w1 - w0) / kPi * w[n + M])
                               : static_cast<float>((std::sin(n * w1) - std::sin(n * w0)) / (n * kPi) * w[n + M]);
    double pk = taps[M];
    for (int n = 1; n <= M; n++) pk += 2 * taps[n + M] * std::cos(n * (w0 + w1) * 0.5);
    gain /= pk;
    for (auto& t : taps) t = static_cast<float>(t * gain);
    return taps;
}
inline std::vector<float> band_pass(double gain, double fs, double lo, double hi, double tw, int win = WIN_HAMMING)
{ return band_pass_core(gain, fs, lo, hi, ntaps_for_window(fs, tw, win), win); }
inline std::vector<float> band_pass_2(double gain, double fs, double lo, double hi, double tw, double att, int win = WIN_HAMMING)
{ return band_pass_core(gain, fs, lo, hi, ntaps_for_attenuation(fs, tw, att), win); }

// complex band-pass: real low-pass prototype spun to the band centre; returns interleaved (re,im)
inline std::vector<float> complex_band_pass_core(double gain, double fs, double lo, double hi, int ntaps, int win)
{
    std::vector<float> lp = low_pass_core(gain, fs, (hi - lo) / 2, ntaps, win), out(2 * ntaps);
    const float freq = static_cast<float>(kPi * (hi + lo) / fs);
    float phase = (ntaps & 1) ? -freq * static_cast<float>(ntaps >> 1) : -freq / 2.0f * static_cast<float>((1 + 2 * ntaps) >> 1);
    for (int i = 0; i < ntaps; i++) {
        out[2 * i] = lp[i] * cosf(phase);
        out[2 * i + 1] = lp[i] * sinf(phase);
        phase += freq;
    }
    return out;
}
inline std::vector<float> complex_band_pass(double gain, double fs, double lo, double hi, double tw, int win = WIN_HAMMING)
{ return complex_band_pass_core(gain, fs, lo, hi, ntaps_for_window(fs, tw, win), win); }
inline std::vector<float> complex_band_pass_2(double gain, double fs, double lo, double hi, double tw, double att, int win = WIN_HAMMING)
{ return complex_band_pass_core(gain, fs, lo, hi, ntaps_for_attenuation(fs, tw, att), win); }

// gr::filter::firdes::gaussian (gr_mod_gmsk.cpp:77-79)
inline std::vector<float> gaussian(double gain, double spb, double bt, int ntaps)
{
    std::vector<float> taps(ntaps);
    double scale = 0;
    const double dt = 1.0 / spb;
    const double s = 1.0 / (std::sqrt(std::log(2.0)) / (2 * kPi * bt));
    double t0 = -0.5 * ntaps;
    for (int i = 0; i < ntaps; i++) {
        t0++;
        const double ts = s * dt * t0;
        taps[i] = static_cast<float>(std::exp(-0.5 * ts * ts));
        scale += taps[i];
    }
    for (int i = 0; i < ntaps; i++) taps[i] = static_cast<float>(taps[i] / scale * gain);
    return taps;
}

inline std::vector<float> root_raised_cosine(double gain, double fs, double symrate, double alpha, int ntaps)
{
    ntaps |= 1;
    const double spb = fs / symrate;
    std::vector<float> taps(ntaps);
    double sum = 0;
    for (int i = 0; i < ntaps; i++) {
        const double x = i - ntaps / 2;
        const double x1 = kPi * x / spb;
        double x2 = 4 * alpha * x / spb;
        double x3 = x2 * x2 - 1;
        double num, den;
        if (std::fabs(x3) >= 0.000001) {
            num = (i != ntaps / 2) ? std::cos((1 + alpha) * x1) + std::sin((1 - alpha) * x1) / (4 * alpha * x / spb)
                                   : std::cos((1 + alpha) * x1) + (1 - alpha) * kPi / (4 * alpha);
            den = x3 * kPi;
        } else {
            if (alpha == 1) { taps[i] = -1; sum += taps[i]; continue; }
            x3 = (1 - alpha) * x1;
            x2 = (1 + alpha) * x1;
            num = (std::sin(x2) * (1 + alpha) * kPi - std::cos(x3) * ((1 - alpha) * kPi * spb) / (4 * alpha * x)
                   + std::sin(x3) * spb * spb / (4 * alpha * x * x));
            den = -32 * kPi * alpha * alpha * x / spb;
        }
        taps[i] = static_cast<float>(4 * alpha * num / den);
        sum += taps[i];
    }
    for (auto& t : taps) t = static_cast<float>(t * gain / sum);
    return taps;
}

// FM de-emphasis / pre-emphasis one-pole sections (bilinear transform; the corner is pre-warped with
// the single-precision tanf exactly as the reference's emphasis.cpp:28,66-67 does)
inline void deemph_taps(int fs_i, double tau, double a[2], double b[2])
{
    const double fs = fs_i;
    const double w_ca = 2.0 * fs * tanf(static_cast<float>((1.0 / tau) / (2.0 * fs)));
    const double k = -w_ca / (2.0 * fs);
    const double p1 = (1.0 + k) / (1.0 - k);
    const double b0 = -k / (1.0 - k);
    b[0] = b0; b[1] = b0 * 1.0;
    a[0] = 1.0; a[1] = -p1;
}
inline void preemph_taps(int fs_i, double tau, double fh, double a[2], double b[2])
{
    const double fs = fs_i;
    if (fh <= 0.0 || fh >= fs / 2.0) fh = 0.925 * fs / 2.0;
    const double w_cla = 2.0 * fs * tanf(static_cast<float>((1.0 / tau) / (2.0 * fs)));
    const double w_cha = 2.0 * fs * tanf(static_cast<float>((2.0 * kPi * fh) / (2.0 * fs)));
    const double kl = -w_cla / (2.0 * fs), kh = -w_cha / (2.0 * fs);
    const double z1 = (1.0 + kl) / (1.0 - kl), p1 = (1.0 + kh) / (1.0 - kh), b0 = (1.0 - kl) / (1.0 - kh);
    const double g = std::fabs(1.0 - p1) / (b0 * std::fabs(1.0 - z1));
    b[0] = g * b0; b[1] = g * b0 * -z1;
    a[0] = 1.0; a[1] = -p1;
}

// ---- lookup tables used by the device code
// gr::fast_atan2f: atan(i/255) as the 7-significant-digit literals GNU Radio's table holds
inline std::vector<float> atan_table()
{
    std::vector<float> t(257);
    char buf[64];
    for (int i = 0; i < 256; i++) { std::snprintf(buf, sizeof buf, "%e", std::atan(i / 255.0)); t[i] = std::strtof(buf, nullptr); }
    t[256] = t[255];
    return t;
}
// gr::blocks::tanhf_lut
inline std::vector<float> tanh_table()
{
    std::vector<float> t(256);
    for (int i = 0; i < 256; i++) t[i] = static_cast<float>(std::tanh((i - 128) / 64.0));
    return t;
}
// gr::fxpt sine table: (slope, intercept) of sin over u = (Q32 phase)>>1
inline std::vector<float> fxpt_sine_table()
{
    std::vector<float> t(2048);
    const double scale = kPi / 1073741824.0, inc = 2097152.0;
    for (int i = 0; i < 1024; i++) {
        const double a = i * inc, b = (i + 1) * inc;
        const double m = (std::sin(b * scale) - std::sin(a * scale)) / (b - a);
        t[2 * i] = static_cast<float>(m);
        t[2 * i + 1] = static_cast<float>(std::sin(a * scale) - m * a);
    }
    return t;
}
// MMSE 8-tap fractional-delay bank (129 phases), band limit 0.25 fs, 6 significant digits
inline std::vector<float> mmse_table()
{
    auto s = [](double d) { return std::fabs(d) < 1e-12 ? 0.5 : std::sin(2 * kPi * 0.25 * d) / (kPi * d); };
    std::vector<float> t(129 * 8);
    char buf[64];
    for (int imu = 0; imu <= 128; imu++) {
        const double mu = imu / 128.0;
        double A[8][9];
        for (int a = 0; a < 8; a++) {
            for (int b = 0; b < 8; b++) A[a][b] = s(static_cast<double>(a - b));
            A[a][8] = s(static_cast<double>(a - 4) + mu);
        }
        for (int c = 0; c < 8; c++) {   // Gaussian elimination, partial pivoting
            int p = c;
            for (int r = c + 1; r < 8; r++) if (std::fabs(A[r][c]) > std::fabs(A[p][c])) p = r;
            if (p != c) for (int k = 0; k < 9; k++) { double tmp = A[c][k]; A[c][k] = A[p][k]; A[p][k] = tmp; }
            for (int r = c + 1; r < 8; r++) {
                const double f = A[r][c] / A[c][c];
                for (int k = c; k < 9; k++) A[r][k] -= f * A[c][k];
            }
        }
        for (int r = 7; r >= 0; r--) {
            double acc = A[r][8];
            for (int k = r + 1; k < 8; k++) acc -= A[r][k] * A[k][8];
            A[r][8] = acc / A[r][r];
        }
        for (int k = 0; k < 8; k++) {
            double v = A[k][8];
            if (std::fabs(v) < 1e-9) v = 0.0;
            std::snprintf(buf, sizeof buf, "%.5e", v);
            t[imu * 8 + k] = std::strtof(buf, nullptr);
        }
    }
    return t;
}

// digital::clock_tracking_loop gains
inline void clock_loop_gains(float loop_bw, float zeta, float ted_gain, float& alpha, float& beta)
{
    const float k0 = 2.0f / ted_gain;
    const float k1 = expf(-zeta * loop_bw);
    const float sh = sinhf(zeta * loop_bw);
    float cx;
    if (zeta > 1.0f) cx = coshf(loop_bw * sqrtf(zeta * zeta - 1.0f));
    else if (zeta == 1.0f) cx = 1.0f;
    else cx = cosf(loop_bw * sqrtf(1.0f - zeta * zeta));
    alpha = k0 * k1 * sh;
    beta = k0 * (1.0f - k1 * (sh + cx));
}
// blocks::control_loop gains (critically damped, zeta = sqrt(2)/2)
inline void control_loop_gains(float loop_bw, float& alpha, float& beta)
{
    const float damping = sqrtf(2.0f) / 2.0f;
    const float denom = static_cast<float>(1.0 + 2.0 * damping * loop_bw + loop_bw * loop_bw);
    alpha = (4 * damping * loop_bw) / denom;
    beta = (4 * loop_bw * loop_bw) / denom;
}

}  // namespace qrl
