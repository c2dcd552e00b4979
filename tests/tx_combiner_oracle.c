/*
 * tx_combiner_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE ONLY) of the transmit combiner: N modulators -> one SDR stream.
 *
 * Built on its own by tests/tx_combiner_oracle.py.  It compiles tests/tx_frontend_oracle.c (and through it oracle/qrl_oracle.c) into
 * the same translation unit, so the interpolator below is that file's gr_mod_base interpolator unchanged.  The product (qradiolink_b200/)
 * never links, imports or calls it.
 */
#include "tx_frontend_oracle.c"

/* ------------------------------------------------------------------ gr_mod_mmdvm_multi's wiring at SDR rates
 * gr_mod_mmdvm_multi.cpp:53-125, with gr_mod_base's interpolator (gr_mod_base.cpp:38,211-259) as the per-channel resampler:
 *   u_c = qo_tx_frontend at offset 0 (x N, N = samp_rate / 1e6; identity at N = 1)
 *   r_c[n] = u_c[n] e^{j theta_c(n_abs)}: the Q32 NCO of qo_tx_frontend at the DEVICE rate, inc = rint(+offset / samp_rate * 2^32);
 *            a retune is phase-continuous from the next output sample; a channel with inc == base == 0 is not rotated
 *   S      = add_cc in blocks of 8: s_b = ((r_8b + r_8b+1) + ...) + r_8b+7, then S = ((s_0 + s_1) + ...)
 *   y      = (S * (1.0f / C)) * gain per component (multiply_const_cc(1 / num_channels), multiply_const_cc(bb_gain)) */
#define QO_TXC_BLOCK 8
struct qo_tx_combiner_ch { qo_tx_frontend* fe; uint32_t inc, base; long long nbase; };
typedef struct qo_tx_combiner { int samp_rate, N, C; float gain; long long n_out; struct qo_tx_combiner_ch* ch; } qo_tx_combiner;

qo_tx_combiner* qo_tx_combiner_create(int samp_rate, int n_channels)
{
    if (samp_rate < 1000000 || samp_rate > 32000000 || samp_rate % 1000000 || n_channels <= 0) return NULL;
    qo_tx_combiner* t = (qo_tx_combiner*)calloc(1, sizeof *t);
    t->samp_rate = samp_rate; t->N = samp_rate / 1000000; t->C = n_channels; t->gain = 1.0f;
    t->ch = (struct qo_tx_combiner_ch*)calloc((size_t)n_channels, sizeof *t->ch);
    for (int c = 0; c < n_channels; c++) t->ch[c].fe = qo_tx_frontend_create(samp_rate);
    return t;
}
void qo_tx_combiner_destroy(qo_tx_combiner* t)
{
    if (!t) return;
    for (int c = 0; c < t->C; c++) qo_tx_frontend_destroy(t->ch[c].fe);
    free(t->ch);
    free(t);
}
int qo_tx_combiner_ntaps(const qo_tx_combiner* t) { return qo_tx_frontend_ntaps(t->ch[0].fe); }
/* channel < 0: every channel */
void qo_tx_combiner_set_carrier_offset(qo_tx_combiner* t, int channel, double offset_hz)
{
    for (int c = 0; c < t->C; c++) {
        if (channel >= 0 && c != channel) continue;
        struct qo_tx_combiner_ch* k = &t->ch[c];
        k->base = k->base + k->inc * (uint32_t)(t->n_out - k->nbase);
        k->nbase = t->n_out;
        k->inc = (uint32_t)(int32_t)(long long)rint(offset_hz / t->samp_rate * 4294967296.0);
    }
}
void qo_tx_combiner_set_gain(qo_tx_combiner* t, float gain) { t->gain = gain; }
/* iq: C rows of n gr_complex at 1 Msps, row c at iq + 2 c stride; returns the N n summed samples written to out (cap items) */
long qo_tx_combiner_work(qo_tx_combiner* t, const float* iq, long n, long stride, float* out, long cap)
{
    const long m = n * t->N;
    float* u = (float*)malloc(sizeof(float) * 2 * (size_t)(m > 0 ? m : 1));
    float* blk = (float*)calloc(2 * (size_t)(m > 0 ? m : 1), sizeof(float));
    float* S = (float*)calloc(2 * (size_t)(m > 0 ? m : 1), sizeof(float));
    for (int c = 0; c < t->C; c++) {
        struct qo_tx_combiner_ch* k = &t->ch[c];
        qo_tx_frontend_work(k->fe, iq + 2 * (size_t)c * (size_t)stride, n, u, m);
        const int rot = k->inc != 0 || k->base != 0;
        for (long i = 0; i < m; i++) {
            float xr = u[2 * i], xi = u[2 * i + 1];
            if (rot) {
                uint32_t ph = k->base + k->inc * (uint32_t)(t->n_out + i - k->nbase);
                float ang = (float)((double)(int32_t)ph * (M_PI / 2147483648.0));
                float sn, cs; qo_sincosf(ang, &sn, &cs);
                float yr = xr * cs - xi * sn, yi = xr * sn + xi * cs;
                xr = yr; xi = yi;
            }
            if (c % QO_TXC_BLOCK == 0) { blk[2 * i] = xr; blk[2 * i + 1] = xi; }
            else { blk[2 * i] = blk[2 * i] + xr; blk[2 * i + 1] = blk[2 * i + 1] + xi; }
        }
        if (c % QO_TXC_BLOCK == QO_TXC_BLOCK - 1 || c == t->C - 1) {
            for (long i = 0; i < 2 * m; i++) S[i] = c < QO_TXC_BLOCK ? blk[i] : S[i] + blk[i];
        }
    }
    const float g1 = 1.0f / (float)t->C, g2 = t->gain;
    long w = m < cap ? m : cap;
    for (long i = 0; i < w; i++) {
        float yr = S[2 * i], yi = S[2 * i + 1];
        yr = yr * g1; yi = yi * g1; yr = yr * g2; yi = yi * g2;
        out[2 * i] = yr; out[2 * i + 1] = yi;
    }
    t->n_out += m;
    free(u); free(blk); free(S);
    return w;
}
