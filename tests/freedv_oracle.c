/*
 * freedv_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE ONLY) of the FreeDV chains up to the codec2 modem boundary.
 *
 * Built on its own by tests/freedv_oracle.py: it compiles the whole of oracle/qrl_oracle.c into the same translation unit, so the
 * FreeDV chains below reuse that file's restatements (rational resampler with its parity order, direct-form complex filter, firdes,
 * rotator arithmetic) unchanged.  The product (qradiolink_b200/) never links, imports or calls it.
 */
#include "../oracle/qrl_oracle.c"

/* ------------------------------------------------------------------ FreeDV up to the codec2 modem boundary
 * gr_demod_freedv.cpp:31-81 and gr_mod_freedv.cpp:27-85 (instances gr_demod_base.cpp:229-249, gr_mod_base.cpp:181-203) with
 * gr::vocoder::freedv_rx_ss / freedv_tx_ss cut out: those wrap libcodec2, which is not part of the reference.
 * RX: rotator -> rational_resampler_ccf(1, sps, low_pass(sps, fs, 4000, 4000, BH)) (DC gain sps) -> fft_filter_ccc(complex_band_pass_2(1,
 *     8000, lo, fw, 200, 90, BH); LSB: (-fw, -lo)) -> [port 0] -> complex_to_real -> agc2_ff(1e-1, 1e-3, 0.5, 1; max gain 65536) ->
 *     fft_filter_fff(band_pass_2(1, 8000, 200, 3500, 200, 90, BH)) -> x0.1 -> float_to_short(1, 32768) -> [port 1: int16 modem samples,
 *     what freedv_rx_ss consumes].  The feedforward_agc_cc the constructor makes (:56) is never connected.
 * TX: int16 modem samples (what freedv_tx_ss produces) -> short_to_float(1, 32765) -> float_to_complex -> fft_filter_ccc(
 *     complex_band_pass_2(1, 8000, lo, fw, 250, 90, BH); LSB (-fw, -lo)) -> feedforward_agc_cc(512, 1) -> rational_resampler_ccf(sps, 1,
 *     low_pass(sps, fs, fw, 1200, Hamming)) -> x0.98 -> x bb_gain.  _agc and _audio_gain are never connected.
 * float_to_short / short_to_float as for MMDVM in oracle/qrl_oracle.c: x scale, clip, rintf / x (float)(1 / scale). */

/* analog::feedforward_agc_cc(N, ref) of GNU Radio 3.10 (gr-analog feedforward_agc_cc_impl.cc; not in the reference: restated, parity
 * unpinned): history N, y[n] = (ref / max(1e-4, max_{k = n-N+1..n} env(x[k]))) * x[n-N+1], env(z) = max(|re|, |im|), zero history.
 * The output is delayed by N - 1 items and the gain looks ahead over that delay. */
typedef struct { int N; float ref; qvec in; } ffagc_t;
static void ffagc_init(ffagc_t* a, int N, float ref) { a->N = N; a->ref = ref; qv_init(&a->in, 8); qv_push_zero(&a->in, (size_t)(N - 1)); }
static void ffagc_free(ffagc_t* a) { qv_free(&a->in); }
static void ffagc_work(ffagc_t* a, const float* x, size_t n, qvec* out)
{
    qv_push(&a->in, x, n);
    const float* b = (const float*)a->in.d;
    size_t i = 0;
    for (; i + (size_t)a->N <= a->in.n; i++) {
        float m = 1e-4f;
        for (int j = 0; j < a->N; j++) {
            const float re = fabsf(b[2 * (i + j)]), im = fabsf(b[2 * (i + j) + 1]);
            const float e = re > im ? re : im;
            if (e > m) m = e;
        }
        const float g = a->ref / m;
        qv_pushc(out, b[2 * i] * g, b[2 * i + 1] * g);
    }
    qv_drop(&a->in, i);
}
long qo_feedforward_agc_run(const float* in_c, long n, int N, float ref, long chunk, float* out_c)
{
    ffagc_t a; ffagc_init(&a, N, ref);
    qvec o; qv_init(&o, 8);
    if (chunk <= 0) chunk = n > 0 ? n : 1;
    for (long s = 0; s < n; s += chunk) ffagc_work(&a, in_c + 2 * s, (size_t)(n - s < chunk ? n - s : chunk), &o);
    memcpy(out_c, o.d, 8 * o.n);
    const long m = (long)o.n;
    qv_free(&o); ffagc_free(&a);
    return m;
}

static inline short freedv_float_to_short(float v, float scale)
{
    v = v * scale;
    if (v > 32767.0f) v = 32767.0f; else if (v < -32768.0f) v = -32768.0f;
    return (short)rintf(v);
}

typedef struct qo_freedv_rx qo_freedv_rx;
typedef struct qo_freedv_tx qo_freedv_tx;
struct qo_freedv_rx {
    resamp_t rs; fircc_t sbf; resamp_t audio;
    float attack, decay, ref, gain, max_gain;
    uint32_t rot_inc, rot_base; long long rot_nbase, rot_n;
    int samp_rate;
    qvec s_rot, s_res, s_agc, s_aud, port0, port1;
    float taps[3][2 * 4096]; int ntaps[3];
};
qo_freedv_rx* qo_freedv_rx_create(int sps, int samp_rate, int filter_width, int low_cutoff, int sb)
{
    if (sps <= 0 || samp_rate / sps != 8000 || low_cutoff < 0 || low_cutoff >= filter_width || filter_width > 4000) return NULL;
    qo_freedv_rx* r = (qo_freedv_rx*)calloc(1, sizeof *r);
    r->samp_rate = samp_rate;
    r->ntaps[0] = qo_firdes_low_pass(sps, samp_rate, 4000, 4000, QO_WIN_BLACKMAN_HARRIS, r->taps[0], 2 * 4096);
    resamp_init(&r->rs, 2, 1, sps, r->taps[0], r->ntaps[0]);
    r->ntaps[1] = sb ? qo_firdes_complex_band_pass_2(1, 8000, -filter_width, -low_cutoff, 200, 90, QO_WIN_BLACKMAN_HARRIS, r->taps[1], 4096)
                     : qo_firdes_complex_band_pass_2(1, 8000, low_cutoff, filter_width, 200, 90, QO_WIN_BLACKMAN_HARRIS, r->taps[1], 4096);
    fircc_init(&r->sbf, r->taps[1], r->ntaps[1]);
    r->ntaps[2] = qo_firdes_band_pass_2(1, 8000, 200, 3500, 200, 90, QO_WIN_BLACKMAN_HARRIS, r->taps[2], 2 * 4096);
    resamp_init(&r->audio, 1, 1, 1, r->taps[2], r->ntaps[2]);
    r->attack = 1e-1f; r->decay = 1e-3f; r->ref = 0.5f; r->gain = 1.0f; r->max_gain = 65536.0f;
    qv_init(&r->s_rot, 8); qv_init(&r->s_res, 8); qv_init(&r->s_agc, 4); qv_init(&r->s_aud, 4);
    qv_init(&r->port0, 8); qv_init(&r->port1, 2);
    return r;
}
void qo_freedv_rx_destroy(qo_freedv_rx* r)
{
    if (!r) return;
    resamp_free(&r->rs); fircc_free(&r->sbf); resamp_free(&r->audio);
    qv_free(&r->s_rot); qv_free(&r->s_res); qv_free(&r->s_agc); qv_free(&r->s_aud); qv_free(&r->port0); qv_free(&r->port1);
    free(r);
}
/* gr_demod_freedv::set_agc_attack / set_agc_decay (:85-93); 0 = applied, -1 = no such setter (set_squelch is codec2's) */
int qo_freedv_rx_set_param(qo_freedv_rx* r, int key, double value)
{
    if (key == QO_PARAM_AGC_ATTACK) { r->attack = (float)value; return 0; }
    if (key == QO_PARAM_AGC_DECAY) { r->decay = (float)value; return 0; }
    return -1;
}
void qo_freedv_rx_set_carrier_offset(qo_freedv_rx* r, double offset_hz)
{
    r->rot_base = r->rot_base + r->rot_inc * (uint32_t)(r->rot_n - r->rot_nbase);
    r->rot_nbase = r->rot_n;
    r->rot_inc = (uint32_t)(int32_t)(long long)rint(-offset_hz / r->samp_rate * 4294967296.0);
}
int qo_freedv_rx_work(qo_freedv_rx* r, const float* iq, long T)
{
    const float* x = iq;
    if (r->rot_inc != 0 || r->rot_base != 0) {            /* the rotator of rx_rotate */
        r->s_rot.n = 0;
        for (long i = 0; i < T; i++) {
            uint32_t ph = r->rot_base + r->rot_inc * (uint32_t)(r->rot_n + i - r->rot_nbase);
            float ang = (float)((double)(int32_t)ph * (M_PI / 2147483648.0));
            float sn, cs; qo_sincosf(ang, &sn, &cs);
            qv_pushc(&r->s_rot, iq[2 * i] * cs - iq[2 * i + 1] * sn, iq[2 * i] * sn + iq[2 * i + 1] * cs);
        }
        x = (const float*)r->s_rot.d;
    }
    r->rot_n += T;
    r->s_res.n = 0; resamp_work(&r->rs, x, (size_t)T, &r->s_res);
    const size_t p0 = r->port0.n;
    fircc_work(&r->sbf, (const float*)r->s_res.d, r->s_res.n, &r->port0);
    const float* f = (const float*)r->port0.d + 2 * p0;
    r->s_agc.n = 0;
    for (size_t i = 0; i < r->port0.n - p0; i++) {
        /* complex_to_real, then analog::kernel::agc2_ff::scale (fabsf form, as in the AM chain) */
        const float out = f[2 * i] * r->gain;
        const float tmp = fabsf(out) - r->ref;
        float rate = r->decay;
        if (fabsf(tmp) > r->gain) rate = r->attack;
        r->gain -= tmp * rate;
        if (r->gain < 0.0f) r->gain = 10e-5f;
        if (r->max_gain > 0.0f && r->gain > r->max_gain) r->gain = r->max_gain;
        qv_pushf(&r->s_agc, out);
    }
    r->s_aud.n = 0; resamp_work(&r->audio, (const float*)r->s_agc.d, r->s_agc.n, &r->s_aud);
    const float* a = (const float*)r->s_aud.d;
    for (size_t i = 0; i < r->s_aud.n; i++) {
        const float v = a[i] * 0.1f;                        /* multiply_const_ff(0.1) */
        const short s = freedv_float_to_short(v, 32768.0f);
        qv_push(&r->port1, &s, 1);
    }
    return 0;
}
long qo_freedv_rx_port_items(qo_freedv_rx* r, int port) { return (long)(port == 0 ? r->port0.n : r->port1.n); }
const void* qo_freedv_rx_port_data(qo_freedv_rx* r, int port) { return port == 0 ? (const void*)r->port0.d : (const void*)r->port1.d; }
void qo_freedv_rx_clear(qo_freedv_rx* r) { r->port0.n = 0; r->port1.n = 0; }
/* which: 0 = stage-1 low-pass, 1 = side-band filter (complex: 2 floats per tap), 2 = audio band-pass; returns the tap count */
int qo_freedv_rx_taps(qo_freedv_rx* r, int which, float* out, int cap)
{
    const int n = r->ntaps[which], per = which == 1 ? 2 : 1;
    if (out && n <= cap) memcpy(out, r->taps[which], sizeof(float) * (size_t)(per * n));
    return n;
}

struct qo_freedv_tx {
    fircc_t sbf; ffagc_t agc; resamp_t rs; float bb_gain;
    qvec s_c, s_f, s_g, out;
    float taps[2][2 * 4096]; int ntaps[2];
};
qo_freedv_tx* qo_freedv_tx_create(int sps, int samp_rate, int filter_width, int low_cutoff, int sb)
{
    if (sps <= 0 || samp_rate / sps != 8000 || low_cutoff < 0 || low_cutoff >= filter_width || filter_width > 4000) return NULL;
    qo_freedv_tx* t = (qo_freedv_tx*)calloc(1, sizeof *t);
    t->ntaps[0] = sb ? qo_firdes_complex_band_pass_2(1, 8000, -filter_width, -low_cutoff, 250, 90, QO_WIN_BLACKMAN_HARRIS, t->taps[0], 4096)
                     : qo_firdes_complex_band_pass_2(1, 8000, low_cutoff, filter_width, 250, 90, QO_WIN_BLACKMAN_HARRIS, t->taps[0], 4096);
    fircc_init(&t->sbf, t->taps[0], t->ntaps[0]);
    ffagc_init(&t->agc, 512, 1.0f);
    t->ntaps[1] = qo_firdes_low_pass(sps, samp_rate, filter_width, 1200, QO_WIN_HAMMING, t->taps[1], 2 * 4096);
    resamp_init(&t->rs, 2, sps, 1, t->taps[1], t->ntaps[1]);
    t->bb_gain = 1.0f;
    qv_init(&t->s_c, 8); qv_init(&t->s_f, 8); qv_init(&t->s_g, 8); qv_init(&t->out, 8);
    return t;
}
void qo_freedv_tx_destroy(qo_freedv_tx* t)
{
    if (!t) return;
    fircc_free(&t->sbf); ffagc_free(&t->agc); resamp_free(&t->rs);
    qv_free(&t->s_c); qv_free(&t->s_f); qv_free(&t->s_g); qv_free(&t->out);
    free(t);
}
void qo_freedv_tx_set_bb_gain(qo_freedv_tx* t, float g) { t->bb_gain = g; }      /* gr_mod_freedv::set_bb_gain */
int qo_freedv_tx_work(qo_freedv_tx* t, const short* in, long n)
{
    const float inv = (float)(1.0 / 32765.0);
    t->s_c.n = 0;
    for (long i = 0; i < n; i++) qv_pushc(&t->s_c, (float)in[i] * inv, 0.0f);          /* short_to_float, float_to_complex */
    t->s_f.n = 0; fircc_work(&t->sbf, (const float*)t->s_c.d, t->s_c.n, &t->s_f);
    t->s_g.n = 0; ffagc_work(&t->agc, (const float*)t->s_f.d, t->s_f.n, &t->s_g);
    const size_t o0 = t->out.n;
    resamp_work(&t->rs, (const float*)t->s_g.d, t->s_g.n, &t->out);
    float* m = (float*)t->out.d;
    for (size_t i = 2 * o0; i < 2 * t->out.n; i++) { m[i] = m[i] * 0.98f; m[i] = m[i] * t->bb_gain; }
    return 0;
}
long qo_freedv_tx_out_items(qo_freedv_tx* t) { return (long)t->out.n; }
const float* qo_freedv_tx_out_data(qo_freedv_tx* t) { return (const float*)t->out.d; }
void qo_freedv_tx_out_clear(qo_freedv_tx* t) { t->out.n = 0; }
/* which: 0 = side-band filter (complex), 1 = interpolator low-pass */
int qo_freedv_tx_taps(qo_freedv_tx* t, int which, float* out, int cap)
{
    const int n = t->ntaps[which], per = which == 0 ? 2 : 1;
    if (out && n <= cap) memcpy(out, t->taps[which], sizeof(float) * (size_t)(per * n));
    return n;
}

/* The speech side of the vocoder, which stays on the host next to codec2 (definitions for an adapter):
 * RX behind freedv_rx_ss: short_to_float(1, 32768) -> multiply_const_ff(2) */
void qo_freedv_speech_out(const short* in, long n, float* out)
{
    const float inv = (float)(1.0 / 32768.0);
    for (long i = 0; i < n; i++) { float v = (float)in[i] * inv; out[i] = v * 2.0f; }
}
/* TX in front of freedv_tx_ss: fft_filter_fff(band_pass(1, 8000, 200, 3500, 350, BH)) -> float_to_short(1, 32765); one stream from
 * zero history, returns n */
long qo_freedv_speech_in(const float* in, long n, short* out)
{
    static float taps[4096];
    const int nt = qo_firdes_band_pass(1, 8000, 200, 3500, 350, QO_WIN_BLACKMAN_HARRIS, taps, 4096);
    resamp_t f; resamp_init(&f, 1, 1, 1, taps, nt);
    qvec o; qv_init(&o, 4);
    resamp_work(&f, in, (size_t)n, &o);
    const float* a = (const float*)o.d;
    for (size_t i = 0; i < o.n; i++) out[i] = freedv_float_to_short(a[i], 32765.0f);
    const long m = (long)o.n;
    qv_free(&o); resamp_free(&f);
    return m;
}
