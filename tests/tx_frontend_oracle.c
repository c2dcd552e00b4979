/*
 * tx_frontend_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE ONLY) of gr_mod_base's transmit front end: carrier-offset rotator at 1 Msps
 * and x N interpolator to the device rate.
 *
 * Built on its own by tests/tx_frontend_oracle.py: it compiles the whole of oracle/qrl_oracle.c into the same translation unit, so the
 * definition below reuses that file's rational resampler (arm layout, parity order), firdes and sin/cos unchanged.  The product
 * (qradiolink_b200/) never links, imports or calls it.
 */
#include "../oracle/qrl_oracle.c"

/* ------------------------------------------------------------------ gr_mod_base transmit front end
 * gr_mod_base.cpp:38,211-293,530-754,799-805: modulator (1 Msps) -> rotator_cc(2 pi offset / 1e6) -> [samp_rate >= 2 Msps:
 * rational_resampler_ccf(N, 1, low_pass(N, samp_rate, 480000, 20000, BLACKMAN_HARRIS)), N = samp_rate / 1e6] -> SDR sink.
 *   - Rotator: the Q32 NCO of rx_rotate with the opposite sign, inc = rint(+offset / 1e6 * 2^32) (the reference divides by the
 *     default sample_rate of set_carrier_offset, 1e6, not by the device rate); a retune is phase-continuous from the next input
 *     sample on; no rotation while inc == base == 0.
 *   - N = 1: the rotator alone (the reference has no resampler in the graph there).
 *   - N >= 2: resamp_init(2, N, 1): each input sample gives exactly N outputs, y[N m + p] = one fmaf chain per component over the
 *     zero-padded arm p, oldest sample first (resamp_work's order for L > 1). */
struct qo_tx_frontend { int samp_rate, N, ntaps; resamp_t rs; uint32_t inc, base; long long nbase, n; qvec s_rot; };
typedef struct qo_tx_frontend qo_tx_frontend;

qo_tx_frontend* qo_tx_frontend_create(int samp_rate)
{
    if (samp_rate < 1000000 || samp_rate > 32000000 || samp_rate % 1000000) return NULL;
    qo_tx_frontend* f = (qo_tx_frontend*)calloc(1, sizeof *f);
    f->samp_rate = samp_rate; f->N = samp_rate / 1000000;
    if (f->N >= 2) {
        static float T[16384];
        f->ntaps = qo_firdes_low_pass(f->N, samp_rate, 480000, 20000, QO_WIN_BLACKMAN_HARRIS, T, 16384);
        resamp_init(&f->rs, 2, f->N, 1, T, f->ntaps);
    }
    qv_init(&f->s_rot, 8);
    return f;
}
void qo_tx_frontend_destroy(qo_tx_frontend* f)
{
    if (!f) return;
    if (f->N >= 2) resamp_free(&f->rs);
    qv_free(&f->s_rot);
    free(f);
}
/* taps of the interpolator (0 at 1 Msps: no resampler) */
int qo_tx_frontend_ntaps(const qo_tx_frontend* f) { return f->ntaps; }
void qo_tx_frontend_set_carrier_offset(qo_tx_frontend* f, double offset_hz)
{
    f->base = f->base + f->inc * (uint32_t)(f->n - f->nbase);
    f->nbase = f->n;
    f->inc = (uint32_t)(int32_t)(long long)rint(offset_hz / 1e6 * 4294967296.0);
}
/* n input samples at 1 Msps -> returns the samples at samp_rate written to out (complex interleaved, cap items; N n of them) */
long qo_tx_frontend_work(qo_tx_frontend* f, const float* iq, long n, float* out, long cap)
{
    const float* x = iq;
    if (f->inc != 0 || f->base != 0) {
        f->s_rot.n = 0;
        for (long i = 0; i < n; i++) {
            uint32_t ph = f->base + f->inc * (uint32_t)(f->n + i - f->nbase);
            float ang = (float)((double)(int32_t)ph * (M_PI / 2147483648.0));
            float sn, cs; qo_sincosf(ang, &sn, &cs);
            float xr = iq[2 * i], xi = iq[2 * i + 1];
            qv_pushc(&f->s_rot, xr * cs - xi * sn, xr * sn + xi * cs);
        }
        x = (const float*)f->s_rot.d;
    }
    f->n += n;
    if (f->N == 1) {
        long m = n < cap ? n : cap;
        memcpy(out, x, (size_t)m * 8);
        return m;
    }
    qvec o; qv_init(&o, 8);
    resamp_work(&f->rs, x, (size_t)n, &o);
    long m = (long)o.n < cap ? (long)o.n : cap;
    memcpy(out, o.d, (size_t)m * 8);
    qv_free(&o);
    return m;
}
