/*
 * qrl_b200.h -- C ABI of libqrl_b200.so: batched-channel, H100-native replacements for the per-mode
 * GNU Radio hier-blocks that QRadioLink's gr_demod_base / gr_mod_base connect between the SDR
 * source/sink and the gr_*_sink / gr_*_source boundary blocks.
 *
 * Every entry point returns 0 on success or a negative QRL_E* code; no C++ exception crosses the ABI.
 * qrl_last_error() gives the message for the last failure on a handle (or the process-wide one for
 * create failures when handle == NULL).  One caller thread per handle (same contract as a GNU Radio
 * block's work(): /root/reference/src/gr/gr_bit_sink.h:36-38).
 *
 * What each entry point replaces in the reference:
 *   qrl_rx_create      make_gr_demod_nbfm / make_gr_demod_4fsk / make_gr_demod_qpsk ... factories
 *                      (src/gr/gr_demod_4fsk.h:51-53, gr_demod_qpsk.h:48-50, gr_demod_nbfm.h:38-39) as
 *                      instantiated by gr_demod_base.cpp:203-228, for n_channels independent channels.
 *   qrl_rx_work        the flattened hier-block's work()/general_work() calls for one chunk of the
 *                      1 Msps gr_complex stream (gr_demod_base.cpp:180 "demod_valve" -> hier block),
 *                      including the rotator_cc carrier shift (gr_demod_base.cpp:57,1220-1225).
 *   qrl_rx_read_port   what gr_const_sink / gr_audio_sink / gr_bit_sink (src/gr/gr_bit_sink.cpp:45-84,
 *                      gr_audio_sink.cpp:49-90) receive on output ports 0..3 of the hier block.
 *   qrl_rx_set_param   set_squelch / set_filter_width / set_agc_attack ... (gr_demod_nbfm.h:47-49).
 *   qrl_tx_create/work make_gr_mod_4fsk ... (src/gr/gr_mod_4fsk.h:46-48; gr_mod_base.cpp:155-180) fed by
 *                      gr_byte_source (src/gr/gr_byte_source.cpp:54-106).
 */
#ifndef QRL_B200_H
#define QRL_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QRL_OK 0
#define QRL_EINVAL (-22)      /* bad argument / unsupported mode */
#define QRL_ENOMEM (-12)
#define QRL_ECUDA (-5)        /* CUDA runtime error, see qrl_last_error */
#define QRL_ERANGE (-34)      /* chunk larger than the handle was created for */
#define QRL_ENODEV (-19)      /* no CUDA device: this library has no CPU fallback */

/* hier-block kinds: one per reference file src/gr/gr_demod_<x>.cpp / gr_mod_<x>.cpp */
enum qrl_kind {
    QRL_DEMOD_NBFM = 1, QRL_DEMOD_4FSK = 2, QRL_DEMOD_QPSK = 3, QRL_DEMOD_BPSK = 4, QRL_DEMOD_2FSK = 5,
    QRL_DEMOD_SSB = 6,
    QRL_DEMOD_AM = 7,         /* gr_demod_am.cpp:28-82 (SURVEY 8f row 3); ports: IQ, float audio at 8 ksps */
    QRL_DEMOD_M17 = 10,       /* gr_demod_m17.cpp:30-113 (SURVEY 8f row 3); ports: IQ at 24 ksps, symbols, hard bits (2 per symbol) */
    QRL_DEMOD_DMR = 11,       /* gr_demod_dmr.cpp:32-112 (SURVEY 8f row 3); qrl_rx_create ignores carrier_freq / filter_width / flag; ports: IQ at
                                 24 ksps, symbols, hard bits (2 per symbol), FLOAT symbol filter output (one per port-0 sample) */
    QRL_DEMOD_DSSS = 12,      /* gr_demod_dsss.cpp:32-124 (SURVEY 8f row 3; make_gr_demod_dsss(25, 1e6, 1700, 150)): Barker-13 BPSK at 16 symbols/s;
                                 ports: IQ at 5200 sps, symbols, decoded bits of the two decoders (4 ports like BPSK).  The despreader's
                                 look-back beyond its declared history is DEFINED as the stream's own older items (zeros at the start) */
    QRL_DEMOD_WBFM = 9,       /* gr_demod_wbfm.cpp:28-70 (SURVEY 8f row 3); ports: IQ at 200 ksps, float audio at 8 ksps */
    QRL_DEMOD_GMSK = 8,       /* gr_demod_gmsk.cpp:30-134 (SURVEY 8f row 3); sps 10 / 5 / 1 = GMSK1K / 2K / 10K; 4 ports like 2FSK */
    QRL_DEMOD_FREEDV = 13,    /* gr_demod_freedv.cpp:31-81 up to the input of freedv_rx_ss (codec2 runs on the host): created with
                                 qrl_rx_create_freedv.  Ports: 0 = IQ at 8 ksps (sps x the input level: the stage-1 low-pass has a DC gain of
                                 sps, the reference's taps); 1 = INT16 modem samples at 8 ksps (item size 2), the float_to_short(1, 32768)
                                 output that freedv_rx_ss consumes -- unlike the reference's port 1, which is float speech behind the vocoder */
    QRL_MOD_4FSK = 101, QRL_MOD_QPSK = 102, QRL_MOD_NBFM = 103, QRL_MOD_BPSK = 104, QRL_MOD_2FSK = 105,
    QRL_MOD_SSB = 106,
    QRL_MOD_GMSK = 107,       /* gr_mod_gmsk.cpp:30-100 (sps 50 / 100 / 10 = GMSK2K / 1K / 10K) */
    QRL_MOD_M17 = 108,        /* gr_mod_m17.cpp:30-95 (sps = 125: x125 / 3 from 24 ksps); items: frame bytes, 4 symbols each */
    QRL_MOD_DSSS = 110,       /* gr_mod_dsss.cpp:27-93 (make_gr_mod_dsss(25, 1e6, 1700, 200), gr_mod_base.cpp:170): one input byte = 208 chips = 10^6 output items, so
                                 max_items is small (the output buffer holds max_items x 8 MB per channel) */
    QRL_MOD_AM = 111,         /* gr_mod_am.cpp:25-72 (make_gr_mod_am(125, 1e6, 1700, 5000), gr_mod_base.cpp:167): float audio at 8 ksps in, like NBFM / SSB */
    QRL_MOD_FREEDV = 112,     /* gr_mod_freedv.cpp:27-85 behind freedv_tx_ss: created with qrl_tx_create_freedv; items: int16 modem samples at
                                 8 ksps (what freedv_tx_ss produces), sps gr_complex outputs per item in every call */
    QRL_MOD_DMR = 109         /* gr_mod_dmr.cpp:27-93 (the M17 modulator's structure with the DMR pulse, deviation 0.85 and
                                 gr_zero_idle_bursts in place of the IF low-pass; see qrl_tx_zero_samples) */
};

/* runtime parameters (qrl_rx_set_param / qrl_tx_set_param) */
enum qrl_param {
    QRL_PARAM_CARRIER_OFFSET_HZ = 1,  /* rotator_cc phase increment, gr_demod_base.cpp:1220-1225 */
    QRL_PARAM_SQUELCH_DB = 2,         /* gr_demod_nbfm::set_squelch */
    QRL_PARAM_FILTER_WIDTH = 3,       /* set_filter_width of gr_demod_nbfm / _ssb / _am / _wbfm (gr_demod_nbfm.cpp:82-90, gr_demod_ssb.cpp:89-101, ...);
                                         through qrl_tx_set_param: gr_mod_nbfm / _ssb / _am::set_filter_width (gr_mod_nbfm.cpp:78-93, gr_mod_ssb.cpp:85-100,
                                         gr_mod_am.cpp:75-85), mid-stream */
    QRL_PARAM_BB_GAIN = 4,            /* gr_mod_*::set_bb_gain */
    QRL_PARAM_CTCSS = 7,              /* gr_demod_nbfm::set_ctcss (gr_demod_nbfm.cpp:97-121): 0 = no tone squelch; f = analog::ctcss_squelch_ff(8000, f, 0.01,
                                         8000, 160, gate) in front of the audio filter (the audio stream shrinks while the tone is absent);
                                         through qrl_tx_set_param: gr_mod_nbfm::set_ctcss (gr_mod_nbfm.cpp:101-139) */
    QRL_PARAM_AGC_ATTACK = 8,         /* gr_demod_ssb::set_agc_attack / gr_demod_am::set_agc_attack (gr_demod_ssb.cpp:108-111, gr_demod_am.cpp:94-97) */
    QRL_PARAM_AGC_DECAY = 9,          /* gr_demod_ssb::set_agc_decay / gr_demod_am::set_agc_decay */
    QRL_PARAM_GAIN = 10,              /* gr_demod_ssb::set_gain (gr_demod_ssb.cpp:118-121): the IF gain in front of the side-band filter */
    QRL_PARAM_RSSI = 6,               /* 1: keep the RSSI tap of rssi_block.cpp:25-45 on port 0 up to date (read with qrl_rx_rssi).
                                         Whenever it goes from 0 to 1 (the first switch-on, mid-stream or not, and every one after
                                         a switch-off) the tap starts afresh: its values are those of rssi_block constructed at that
                                         moment and fed port 0 from the next qrl_rx_work on. */
    QRL_PARAM_OVERLAP_CALLS = 5       /* 1: the loop / FEC tail of qrl_rx_work call k runs under the parallel stages of call
                                         k+1 (streaming use).  Output ports are double-buffered; the results of a call are
                                         ordered on the caller's stream only after qrl_rx_join (or qrl_rx_sync /
                                         qrl_rx_read_port, which wait on the host).  Supported for 4FSK (fm) blocks. */
};

typedef struct qrl_rx qrl_rx;
typedef struct qrl_tx qrl_tx;

/* library / device */
int  qrl_device_count(void);
const char* qrl_version(void);
const char* qrl_last_error(const void* handle);

/* ---- RX ----
 * kind, sps, samp_rate, carrier_freq, filter_width, flag: exactly the arguments of the reference factory
 *   (flag = `fm` for 4FSK/2FSK, `sb` for SSB, ignored otherwise).
 * n_channels independent channels; max_samples = largest T a single qrl_rx_work call will carry. */
int qrl_rx_create(int kind, int sps, int samp_rate, int carrier_freq, int filter_width, int flag,
                  int n_channels, long max_samples, int device, qrl_rx** out);
/* gr_demod_freedv (make_gr_demod_freedv(sps, samp_rate, carrier_freq, filter_width, low_cutoff, mode, sb), gr_demod_freedv.cpp:31-81;
 * instances gr_demod_base.cpp:229-249) as a QRL_DEMOD_FREEDV handle.  The codec2 `mode` only matters to the vocoder behind port 1 and is not
 * taken here.  QRL_EINVAL unless samp_rate / sps == 8000 and 0 <= low_cutoff < filter_width <= 4000.  Setters: QRL_PARAM_AGC_ATTACK /
 * _DECAY (the agc2_ff rates, :85-93), QRL_PARAM_CARRIER_OFFSET_HZ; QRL_PARAM_SQUELCH_DB is codec2's setting (:95-98) and, like
 * FILTER_WIDTH and OVERLAP_CALLS, returns QRL_EINVAL. */
int qrl_rx_create_freedv(int sps, int samp_rate, int carrier_freq, int filter_width, int low_cutoff, int sb,
                         int n_channels, long max_samples, int device, qrl_rx** out);
int qrl_rx_destroy(qrl_rx* h);
/* run all kernels of this handle on an existing CUDA stream (cudaStream_t); NULL = the handle's own stream */
int qrl_rx_set_stream(qrl_rx* h, void* cuda_stream);
int qrl_rx_set_param(qrl_rx* h, int channel /* -1 = all */, int key, double value);
/* Restart every channel's stream at sample 0; waits for everything the handle has in flight.  Afterwards every port of every call
 * is bit-identical to a handle created with the same arguments and given the settings now in force before its first call.  Those
 * settings are: each channel's carrier offset; squelch, filter width and CTCSS; AGC attack and decay, and the IF gain; RSSI on or
 * off; overlapped calls; the stream set with qrl_rx_set_stream.  Everything carried by the stream restarts: histories, rings, loop
 * states, counts, the rotator phase (0 at the first sample after the reset) and the RSSI window.  Until the next qrl_rx_work,
 * qrl_rx_rssi reads -180 + level. */
int qrl_rx_reset(qrl_rx* h);
/* iq: [n_channels][T] interleaved float (re,im) = gr_complex; channel stride = `stride` complex samples.
 * on_device != 0: iq is a device pointer (already in HBM). Otherwise host memory (pinned or pageable);
 * the copy to the device is part of the call.  Asynchronous on the handle's stream.
 * stride == 0 means ONE stream iq[0 .. T) at the handle's 1 Msps feeds every channel (one SDR, several receivers:
 * gr_demod_mmdvm_multi.cpp:68-123's wiring).  Each channel applies its own QRL_PARAM_CARRIER_OFFSET_HZ rotator.  Channel c's outputs
 * are, bit for bit, what the same handle gives for [n_channels][T] with n_channels identical rows: every port, the port counts and
 * qrl_rx_rssi.  Host input is copied to the device once (T samples), device input is read in place; the same holds for
 * qrl_rx_work_sc16 / _sc8, whose one int pair stream is converted once.  A handle may alternate between shared and per-row calls:
 * each channel's stream continues across the switch. */
int qrl_rx_work(qrl_rx* h, const float* iq, long T, long stride, int on_device);
/* The same call fed with the SDR's wire format: interleaved int16 I/Q (UHD / SoapySDR "sc16": 4 bytes per sample, half the PCIe
 * traffic of gr_complex).  Each component becomes float(v) * scale on the device -- one rounding, the arithmetic of the host-side
 * converter that sits in front of the reference's uhd / osmosdr source blocks (gr_demod_base.cpp:166-196; UHD's sc16 -> fc32
 * scale is 1 / 32767) -- and the chain then runs exactly as qrl_rx_work on that gr_complex stream.  stride in int16 pairs. */
int qrl_rx_work_sc16(qrl_rx* h, const short* iq, long T, long stride, float scale, int on_device);
/* the same for 8-bit front ends (HackRF and other int8 sources of gr-osmosdr, 2 bytes per sample): float(v) * scale, stride in int8 pairs */
int qrl_rx_work_sc8(qrl_rx* h, const signed char* iq, long T, long stride, float scale, int on_device);
/* wait for everything submitted so far */
/* RSSI tap (SURVEY 8f row 4): per channel the value probe_signal_f holds behind rssi_block (|x|^2 -> moving_average(2000) ->
 * single_pole_iir(0.04) -> 10 log10 -> + level; /root/reference/src/gr/rssi_block.cpp:25-45, gr_demod_base.cpp:199-200) after the
 * last qrl_rx_work; rssi_db_host [n_channels]; needs QRL_PARAM_RSSI = 1 */
int qrl_rx_rssi(qrl_rx*, float level, float* rssi_db_host);
/* QRL_PARAM_OVERLAP_CALLS: make the handle's stream wait (on the device, without blocking the host) for everything the
 * calls so far have started; a no-op otherwise */
int qrl_rx_join(qrl_rx*);
int qrl_rx_sync(qrl_rx* h);
/* number of output ports (2 for analog blocks, 3 for 4FSK/QPSK, 4 for BPSK/2FSK) and item size in bytes */
int qrl_rx_num_ports(const qrl_rx* h);
int qrl_rx_port_itemsize(const qrl_rx* h, int port);
/* copy what the last qrl_rx_work call produced on `port` into dst[n_channels][cap] (items), and the
 * per-channel item counts into counts[n_channels].  dst_on_device selects a device destination. Syncs. */
int qrl_rx_read_port(qrl_rx* h, int port, void* dst, long cap, int* counts, int dst_on_device);
/* device-resident view of a port (no copy): pointer to [n_channels][*cap] items and the int counts array */
int qrl_rx_port_device(qrl_rx* h, int port, void** data, long* cap, int** counts);
/* kernels launched by this handle so far (for bench accounting) */
long qrl_rx_launch_count(const qrl_rx* h);
/* per-stage device timing: when enabled, every qrl_rx_work brackets each stage's kernels with CUDA events on
 * the handle's stream.  qrl_rx_profile_read syncs and returns the accumulated milliseconds and launch count of
 * `stage` (0 = stage-1 decimating FIR, 1 = channel filter, 2 = demod/shaping, 3 = loops/symbol sync, 4 = FEC)
 * since the last qrl_rx_profile(h, 1) call. */
/* SM partition in use: SMs reserved for the sequential loop/FEC kernels and SMs left to the parallel stages
 * (both 0 when the driver refused green contexts and plain priority streams are used instead) */
int qrl_rx_sm_partition(const qrl_rx* h, int* loop_sms, int* parallel_sms);
int qrl_rx_profile(qrl_rx* h, int enable);
int qrl_rx_profile_read(qrl_rx* h, int stage, double* ms_total, long* n_launches);

/* ---- TX ---- */
int qrl_tx_create(int kind, int sps, int samp_rate, int carrier_freq, int filter_width, int flag,
                  int n_channels, long max_items, int device, qrl_tx** out);
/* gr_mod_freedv (make_gr_mod_freedv(sps, samp_rate, carrier_freq, filter_width, low_cutoff, mode, sb), gr_mod_freedv.cpp:27-85; instances
 * gr_mod_base.cpp:181-203) as a QRL_MOD_FREEDV handle: qrl_tx_work takes [n_channels][n] int16 modem samples at 8 ksps and produces
 * n x sps gr_complex per channel.  Arguments checked as for qrl_rx_create_freedv; QRL_PARAM_BB_GAIN is the one setter. */
int qrl_tx_create_freedv(int sps, int samp_rate, int carrier_freq, int filter_width, int low_cutoff, int sb,
                         int n_channels, long max_items, int device, qrl_tx** out);
int qrl_tx_destroy(qrl_tx* h);
int qrl_tx_set_stream(qrl_tx* h, void* cuda_stream);
int qrl_tx_set_param(qrl_tx* h, int channel, int key, double value);
/* in: [n_channels][n] bytes (digital), float audio (NBFM / SSB / AM) or int16 modem samples (FreeDV); produces [n_channels][n_out]
 * gr_complex at 1 Msps */
int qrl_tx_work(qrl_tx* h, const void* in, long n, long stride, int on_device);
int qrl_tx_sync(qrl_tx* h);
int qrl_tx_read(qrl_tx* h, float* dst, long cap, long* n_out, int dst_on_device);
int qrl_tx_out_device(qrl_tx* h, float** data, long* stride, long* n_out);
long qrl_tx_launch_count(const qrl_tx* h);
/* QRL_MOD_DMR only: the "zero_samples" stream tag of gr_dmr_source.cpp:148 / gr_mmdvm_source.cpp:264, attached to byte
 * `byte_offset` (absolute position in the channel's input stream since create) with value n_samples; channel = -1: every channel.
 * At gr_zero_idle_bursts (gr_zero_idle_bursts.cpp:45-82) the tag sits on 24 ksps item 20 * byte_offset; `delay` = 62 items earlier
 * the block loads its counter with n_samples and clears one output item per count (a later tag overrides a running count; of two
 * tags on one item the first registered wins).  The block's history also delays the stream by 2 * 720 - 1 items (60 ms).
 * Register a tag before the qrl_tx_work call that feeds byte (byte_offset - 4): a tag whose start item has already been produced
 * clears only what is left of its count.  Deviation from the reference, on purpose: the reference drops a tag that falls into
 * the first 62 items of a scheduler window (its lookup is bounded by the current window); here results do not depend on chunking. */
int qrl_tx_zero_samples(qrl_tx* h, int channel, long long byte_offset, long n_samples);
/* per-stage device timing of the modulator (like qrl_rx_profile): stage 0 = bit chain (scrambler / encoder / mapper),
 * 1 = pulse shaping + frequency modulator, 2 = final interpolating FIR (the HBM-write-bound kernel); FreeDV: 0 = int16 conversion +
 * side-band filter, 1 = feedforward AGC, 2 = x sps interpolator */
int qrl_tx_profile(qrl_tx* h, int enable);
int qrl_tx_profile_read(qrl_tx* h, int stage, double* ms_total, long* n_launches);

/* ---- front end at device rates >= 2 Msps ------------------------------------------------------------------------------------------
 * gr_demod_base::set_samp_rate (/root/reference/src/gr/gr_demod_base.cpp:1303-1362): when the device delivers samp_rate >= 2 Msps the
 * reference puts rational_resampler_ccf(1, samp_rate / 1e6, low_pass(1, samp_rate, 480000, 100000, BLACKMAN_HARRIS)) behind the
 * rotator (which then runs at the device rate, :1220-1225,1358) and in front of the demodulators.  This object is that pair for a batch
 * of channels: [n_channels][T] gr_complex at samp_rate in, [n_channels][T / N] at 1 Msps out -- the device-resident input layout of
 * qrl_rx_work.  Streaming (any chunking), phase-continuous retunes.
 * qrl_frontend_work's stride: >= T, channel c reads iq[c * stride .. c * stride + T).  stride == 0: ONE wideband stream iq[0 .. T) feeds
 * every channel (one SDR, n_channels receivers at their own carrier offsets, gr_demod_mmdvm_multi.cpp:68-123); channel c's output is
 * what [n_channels][T] with n_channels identical rows would give, bit for bit.  Host input is copied to the device once (T samples),
 * device input is read in place.  A handle may alternate between shared and per-channel calls: each channel's stream continues.
 * T > max_in returns QRL_ERANGE; T == 0 returns QRL_OK with no output.
 * samp_rate: a multiple of 1 MHz from 2 to 107 Msps.  Above 107 Msps the /N filter (4517 taps at 108 Msps) and its window no longer fit
 * the decimating kernel's 160 KiB of shared memory, and create returns QRL_EINVAL. */
typedef struct qrl_frontend qrl_frontend;
int  qrl_frontend_create(int samp_rate /* multiple of 1e6, 2e6 .. 107e6 */, int n_channels, long max_in, int device, qrl_frontend** out);
int  qrl_frontend_destroy(qrl_frontend*);
int  qrl_frontend_set_stream(qrl_frontend*, void* cuda_stream);
int  qrl_frontend_set_carrier_offset(qrl_frontend*, int channel /* -1 = all */, double offset_hz);
int  qrl_frontend_work(qrl_frontend*, const float* iq, long T, long stride, int on_device, long* n_out);
int  qrl_frontend_out_device(qrl_frontend*, float** data, long* stride, long* n_out);
int  qrl_frontend_read(qrl_frontend*, float* dst /* [n_channels][cap] gr_complex */, long cap);
long qrl_frontend_launch_count(const qrl_frontend*);

/* ---- transmit front end: carrier offset and x N to the device rate ------------------------------------------------------------------
 * gr_mod_base (src/gr/gr_mod_base.cpp:38,211-293,799-805): every modulator's 1 Msps output goes through rotator_cc(2 pi offset / 1e6)
 * and, when the device runs at samp_rate >= 2 Msps, through rational_resampler_ccf(N, 1, low_pass(N, samp_rate, 480000, 20000,
 * BLACKMAN_HARRIS)) with N = samp_rate / 1e6 (about 210 taps per arm) in front of the SDR sink; at 1 Msps the rotator feeds the sink
 * directly.  This object is that pair for a batch of channels: [n_channels][n] gr_complex at 1 Msps in (host memory, or the device
 * pointer and stride of qrl_tx_out_device on the same device), [n_channels][N n] at samp_rate out.  The rotator divides by 1e6 whatever
 * samp_rate is, as the reference's set_carrier_offset(offset, sample_rate = 1000000) does.  Streaming (any chunking gives the same
 * output, n = 0 is valid), phase-continuous retunes from the next input sample on; channel -1 retunes every channel.
 * qrl_tx_frontend_work returns QRL_ERANGE for n > max_in and QRL_EINVAL for a device pointer of another GPU; the output stays on the
 * device until the next call (qrl_tx_frontend_out_device) or is copied out with qrl_tx_frontend_read.  destroy(NULL) is QRL_OK. */
typedef struct qrl_tx_frontend qrl_tx_frontend;
int  qrl_tx_frontend_create(int samp_rate /* multiple of 1e6, 1e6..32e6 */, int n_channels, long max_in, int device, qrl_tx_frontend** out);
int  qrl_tx_frontend_destroy(qrl_tx_frontend*);
int  qrl_tx_frontend_set_stream(qrl_tx_frontend*, void* cuda_stream);
int  qrl_tx_frontend_set_carrier_offset(qrl_tx_frontend*, int channel /* -1 = all */, double offset_hz);
int  qrl_tx_frontend_work(qrl_tx_frontend*, const float* iq, long n, long stride, int on_device, long* n_out /* N n */);
int  qrl_tx_frontend_out_device(qrl_tx_frontend*, float** data, long* stride, long* n_out);
int  qrl_tx_frontend_read(qrl_tx_frontend*, float* dst /* [n_channels][cap] gr_complex */, long cap);
long qrl_tx_frontend_launch_count(const qrl_tx_frontend*);

/* ---- transmit combiner: N modulators -> one SDR sink ------------------------------------------------------------------------------------
 * gr_mod_mmdvm_multi (src/gr/gr_mod_mmdvm_multi.cpp:53-125) wired for a batch of channels at SDR rates: per channel c, gr_mod_base's
 * interpolator rational_resampler_ccf(N, 1, low_pass(N, samp_rate, 480000, 20000, BLACKMAN_HARRIS)) with N = samp_rate / 1e6 (none at
 * 1 Msps), then rotator_cc(2 pi offset_c / samp_rate) AT THE DEVICE RATE, so a channel can sit anywhere in +-samp_rate / 2; then add_cc
 * over the channels, multiply_const_cc(1 / n_channels) and multiply_const_cc(bb_gain) (default 1).  Out: ONE stream of N n gr_complex.
 *   - rows: a host array of n_channels pointers to n gr_complex each at 1 Msps, 8-byte aligned; all in host memory (on_device = 0,
 *     staged into a [n_channels][max_in] buffer) or all on the handle's device (on_device = 1, read in place: e.g. qrl_tx_out_device's
 *     pointer + c stride, or rows of several modulator handles).  Device rows are read on the combiner's stream: the caller orders
 *     their producers before the call (one shared stream through *_set_stream, or a synchronisation).
 *   - Channels are added in blocks of 8, left to right from each block's first channel, then the block sums left to right: the order
 *     does not depend on chunking or launch shape (with n_channels <= 8 it is add_cc's order).
 *   - Streaming: any chunking gives the same output, n = 0 is valid and gives none.  A carrier-offset change (channel -1 = all) is
 *     phase-continuous from the next output sample; a channel whose rotator never turned (offset 0 since create) is passed unrotated.
 *     A gain change applies from the next call.
 *   - Errors: QRL_EINVAL for a bad samp_rate, channel, a NULL or misaligned row, |offset| > samp_rate / 2, or a device row of another
 *     GPU; QRL_ERANGE for n > max_in.  The output stays on the device until the next work (qrl_tx_combiner_out_device) or is copied out
 *     with qrl_tx_combiner_read.  destroy(NULL) is QRL_OK. */
typedef struct qrl_tx_combiner qrl_tx_combiner;
int  qrl_tx_combiner_create(int samp_rate /* multiple of 1e6, 1e6..32e6 */, int n_channels, long max_in, int device, qrl_tx_combiner** out);
int  qrl_tx_combiner_destroy(qrl_tx_combiner*);
int  qrl_tx_combiner_set_stream(qrl_tx_combiner*, void* cuda_stream);
int  qrl_tx_combiner_set_carrier_offset(qrl_tx_combiner*, int channel /* -1 = all */, double offset_hz /* |f| <= samp_rate / 2 */);
int  qrl_tx_combiner_set_gain(qrl_tx_combiner*, float bb_gain);
int  qrl_tx_combiner_work(qrl_tx_combiner*, const float* const* rows /* host array of n_channels row pointers */, long n, int on_device,
                          long* n_out /* N n */);
int  qrl_tx_combiner_out_device(qrl_tx_combiner*, float** data, long* n_out);   /* one stream, valid until the next work */
int  qrl_tx_combiner_read(qrl_tx_combiner*, float* dst /* cap gr_complex */, long cap);
long qrl_tx_combiner_launch_count(const qrl_tx_combiner*);

/* ---- design helpers (host only; the gr::filter::firdes calls the reference makes at construction /
 *      in set_filter_width, e.g. gr_demod_nbfm.cpp:82-90).  Return tap count or negative error. ---- */
int qrl_firdes_low_pass(double gain, double fs, double fc, double tw, int window, float* out, int cap);
int qrl_firdes_low_pass_2(double gain, double fs, double fc, double tw, double att_db, int window, float* out, int cap);
int qrl_firdes_band_pass(double gain, double fs, double lo, double hi, double tw, int window, float* out, int cap);
int qrl_firdes_complex_band_pass(double gain, double fs, double lo, double hi, double tw, int window, float* out, int cap);
int qrl_firdes_root_raised_cosine(double gain, double fs, double symrate, double alpha, int ntaps, float* out, int cap);
int qrl_firdes_gaussian(double gain, double spb, double bt, int ntaps, float* out, int cap);
int qrl_design_table(const char* name /* "atan","tanh","mmse","fxpt_sine" */, float* out, int cap);
int qrl_design_deemph(int fs, double tau, double* a2, double* b2);

/* ---- polyphase channelizer / synthesizer (SURVEY.md section 8f row 1) -------------------------------------------
 * Replaces gr::filter::pfb_channelizer_ccf::make(M, taps, 1.0) fed by blocks::stream_to_streams(M)
 * (/root/reference/src/gr/gr_demod_mmdvm_multi2.cpp:98-107) and gr::filter::pfb_synthesizer_ccf::make(M, taps, false)
 * (/root/reference/src/gr/gr_mod_mmdvm_multi2.cpp:90-92).  Streaming: history and samples that do not fill a frame
 * of M stay in the handle, results do not depend on chunking.  Channel c of the channelizer is centred on
 * +c*fs/M (ports M/2.. are the negative frequencies, the order both reference wirings rely on,
 * gr_demod_mmdvm_multi2.cpp:110-124).  The channelizer output [M][stride] gr_complex is exactly the device-resident
 * input layout of qrl_rx_work.
 * Commutator / timing (GNU Radio itself is not part of /root/reference, so this is restated, not pinned): with oversample rate 1.0
 * pfb_channelizer_ccf::general_work keeps its filter index at M-1 on every iteration, so stream j (sample x[mM + j] of
 * stream_to_streams) is filtered by branch M-1-j, taps[(M-1-j) + tM], at in[n] for every j and lands in FFT bin M-1-j of a backward
 * (e^{+j...}) FFT: u_k[m] = sum_t taps[k + tM] x[(m-t)M + (M-1-k)], out_c[m] = sum_k u_k[m] e^{+j 2 pi k c / M}.  Output column m
 * therefore needs wideband samples up to mM + M-1: the first column is produced once M samples have arrived.  A caller that
 * assumes a different commutator phase sees the same channels delayed / advanced by up to M-1 WIDEBAND samples (less than one
 * channel-rate sample), which the symbol-timing loops downstream absorb. */
enum { QRL_PFB_CHANNELIZER = 201, QRL_PFB_SYNTHESIZER = 202 };
typedef struct qrl_pfb qrl_pfb;
/* max_in: channelizer = wideband samples per call; synthesizer = columns (samples per channel) per call.
 * Accepted shapes: 1 <= M <= 4096 (4096 channels of 25 kHz = 102.4 Msps) and ceil(ntaps / M) <= 128 taps per branch; M > 4096
 * returns QRL_EINVAL with the limit in qrl_last_error, as does any other bad argument.  M = 10 with 35 taps per branch (the
 * reference's 341-tap prototype) runs register-tiled kernels; every other accepted shape runs a branch-FIR kernel and an
 * exact-order DFT kernel with the intermediate in device memory (about 8 B per wideband sample more of it per handle).
 * Every shape is bit-identical to the oracle's definition: branch FIRs oldest sample first, the DFT as the direct sum over k
 * ascending, both in fmaf. */
int  qrl_pfb_create(int kind, int M, const float* taps, int ntaps, long max_in, int device, qrl_pfb** out);
int  qrl_pfb_destroy(qrl_pfb*);
int  qrl_pfb_set_stream(qrl_pfb*, void* cuda_stream);
/* channelizer: in = n_in wideband gr_complex (in_stride ignored); *n_out = new samples per channel.
 * synthesizer: in = [M][in_stride] gr_complex, n_in columns; *n_out = n_in*M wideband samples.
 * in_on_device = 0: host memory (copied inside the call), 1: device pointer. Asynchronous on the handle's stream. */
int  qrl_pfb_work(qrl_pfb*, const void* in, long n_in, long in_stride, int in_on_device, long* n_out);
int  qrl_pfb_sync(qrl_pfb*);
/* device view of the last call's output: channelizer [M][*stride] gr_complex (*items valid columns),
 * synthesizer [*items] gr_complex; valid until the next qrl_pfb_work */
int  qrl_pfb_out_device(qrl_pfb*, void** data, long* stride, long* items);
/* copy the last call's output to host (channelizer: row c at host_dst + c*dst_stride items) and synchronise */
int  qrl_pfb_read(qrl_pfb*, void* host_dst, long dst_stride);
long qrl_pfb_launch_count(qrl_pfb*);

/* ---- MMDVM multi-channel front end: the per-channel chains either side of the filter bank ------------------------------------------
 * gr_demod_mmdvm_multi2 (/root/reference/src/gr/gr_demod_mmdvm_multi2.cpp:56-126; MMDVM_SAMPLE_RATE 250000, src/config_mmdvm.h:4) behind
 * qrl_pfb's channelizer: for channel c, row rows[c] of the [n_rows][stride] gr_complex slab at 25 ksps (NULL rows = identity; the
 * reference's port map is channels 0..3 on ports 0..3, 4.. on 9, 8, ..) -> rational_resampler_ccf(24, 25, low_pass_2(1, 600k, fw, 2000,
 * 60, BH)) -> low_pass_2(1, 24k, fw, 2000, 60, BH) -> rssi_tag_block (one dB value per 300 items, rssi_tag_block.cpp:42-63) ->
 * quadrature_demod_cf(24000 / (2 pi 12500)) -> x1.0 -> float_to_short(1, 32767): int16 [n_channels][*n_out] at 24 ksps, what
 * gr_mmdvm_sink takes.  No feedback loop anywhere: one thread per item in every stage; results are chunk invariant.
 * gr_mod_mmdvm_multi2 (gr_mod_mmdvm_multi2.cpp:47-126) in front of the synthesizer: int16 [n_channels][n] at 24 ksps -> short_to_float
 * (x (float)(1 / 32767): VOLK's SIMD form) -> x1.0 -> frequency_modulator_fc(2 pi 12500 / 24000) (Q32 phase, as the other modulators) ->
 * low_pass_2(1, 24k, ...) -> x0.8 -> rational_resampler_ccf(25, 24, low_pass_2(25, 600k, ...)) -> rows rows[c] of a zeroed [n_rows][stride]
 * slab at 25 ksps (the synthesizer's input; unused rows are the reference's null_source).  qrl_mmdvm_tx_finish applies what follows
 * the synthesizer, multiply_const_cc(1 / n_channels) and multiply_const_cc(bb_gain), in place on the wideband device buffer.
 * gr_zero_idle_bursts(0) (gr_mod_mmdvm_multi2.cpp:88,108-117; gr_mod_mmdvm.cpp:51-58) = qrl_mmdvm_tx_zero_samples below.
 * Not built: the MMDVM protocol sink / source (ZeroMQ, out of scope). */
typedef struct qrl_mmdvm_rx qrl_mmdvm_rx;
typedef struct qrl_mmdvm_tx qrl_mmdvm_tx;
/* variant 0: the per-channel chains of gr_demod_mmdvm_multi2 / gr_mod_mmdvm_multi2 described above (25 ksps <-> 24 ksps).
 * variant 1: the single-channel blocks gr_demod_mmdvm (gr_demod_mmdvm.cpp:30-64) / gr_mod_mmdvm (gr_mod_mmdvm.cpp:28-70) at
 * MMDVM_SAMPLE_RATE = 250 ksps: rational_resampler_ccf(12, 125, low_pass_2(12, 3 MHz, fw, 2000, 60, BH)), the RSSI tags taken in FRONT of the
 * channel filter, quadrature_demod_cf(24000 / (2 pi 10000)); TX: ... -> x0.8 -> x bb_gain -> rational_resampler_ccf(125, 12) (qrl_mmdvm_tx_finish
 * is not used there); n_channels independent streams are processed at once. */
int  qrl_mmdvm_rx_create(int variant, int n_channels, const int* rows, int n_rows, int filter_width, long max_in, int device, qrl_mmdvm_rx** out);
int  qrl_mmdvm_rx_destroy(qrl_mmdvm_rx*);
int  qrl_mmdvm_rx_set_stream(qrl_mmdvm_rx*, void* cuda_stream);
int  qrl_mmdvm_rx_calibrate_rssi(qrl_mmdvm_rx*, float level);              /* rssi_tag_block::calibrate_rssi */
int  qrl_mmdvm_rx_work(qrl_mmdvm_rx*, const float* iq, long n, long stride, int on_device, long* n_out);
int  qrl_mmdvm_rx_sync(qrl_mmdvm_rx*);
/* device views of the last call: int16 [n_channels][*stride], RSSI dB [n_channels][*rssi_stride] (*n_rssi values, the first one
 * belongs to 24 ksps item *first_rssi_item, the next ones follow every 300 items) */
int  qrl_mmdvm_rx_out_device(qrl_mmdvm_rx*, short** data, long* stride, long* n_out, float** rssi_db, long* rssi_stride, int* n_rssi,
                             long long* first_rssi_item);
int  qrl_mmdvm_rx_read(qrl_mmdvm_rx*, short* dst, long dst_stride, float* rssi_db, long rssi_cap, int* n_rssi, long long* first_rssi_item);
long qrl_mmdvm_rx_launch_count(qrl_mmdvm_rx*);
int  qrl_mmdvm_tx_create(int variant, int n_channels, const int* rows, int n_rows, int filter_width, long max_in, int device, qrl_mmdvm_tx** out);
int  qrl_mmdvm_tx_destroy(qrl_mmdvm_tx*);
int  qrl_mmdvm_tx_set_stream(qrl_mmdvm_tx*, void* cuda_stream);
int  qrl_mmdvm_tx_set_bb_gain(qrl_mmdvm_tx*, float gain);                   /* gr_mod_mmdvm_multi2::set_bb_gain */
/* The "zero_samples" stream tag of gr_mmdvm_source.cpp:264 as gr_zero_idle_bursts(0) consumes it (gr_zero_idle_bursts.cpp:47-86): from item
 * `item_offset` of the zero-idle block's OWN stream on, n_samples outputs of `channel` (-1: all) are cleared; a later tag overrides what is
 * left of a running count; counts carry across calls.  The block's stream is the 24 ksps stream behind the FM modulator for variant 1
 * (gr_mod_mmdvm: every block in front of it is 1:1, so item_offset is the index of the tagged int16 sample) and the 25 ksps stream behind
 * the x25/24 resampler for variant 0 (gr_mod_mmdvm_multi2: GNU Radio's scheduler moves a tag on input sample k across the resampler to item
 * floor(k * 25 / 24 + 1/2); the adapter applies that mapping, qradiolink_b200.mmdvm_tag_item does).  Register a tag before the
 * qrl_mmdvm_tx_work call that produces its item; one registered later clears what is left of its count. */
int  qrl_mmdvm_tx_zero_samples(qrl_mmdvm_tx*, int channel, long long item_offset, long n_samples);
int  qrl_mmdvm_tx_work(qrl_mmdvm_tx*, const short* in, long n, long stride, int on_device, long* n_out);
int  qrl_mmdvm_tx_sync(qrl_mmdvm_tx*);
int  qrl_mmdvm_tx_out_device(qrl_mmdvm_tx*, float** data, long* stride, long* n_out);      /* [n_rows][*stride] gr_complex */
int  qrl_mmdvm_tx_read(qrl_mmdvm_tx*, float* dst, long dst_stride);
int  qrl_mmdvm_tx_finish(qrl_mmdvm_tx*, float* wideband_dev, long n);
long qrl_mmdvm_tx_launch_count(qrl_mmdvm_tx*);

/* ---- display spectrum on the device (SURVEY.md section 8f row 4) -----------------------------------------------------------------
 * rx_fft_c (/root/reference/src/gr/rx_fft.cpp:44-129; gr_demod_base.cpp:166: 32768 points, Blackman-Harris; get_FFT_data :978-986) for
 * n_streams streams at once (the wideband source of a GPU, or every channel of a batch: [n_streams][stride] gr_complex like
 * qrl_rx_work).  One qrl_spectrum_work call is one rx_fft_c::work call: while disabled (the initial state) or while a finished spectrum
 * has not been fetched the whole call is dropped; otherwise samples x window fill the buffer and the first sample AFTER it filled
 * runs the forward FFT and volk_32fc_s32f_power_spectrum_32f(points, fft, N, N) (dB of |X / N|^2).  qrl_spectrum_get copies the points
 * fft-shifted (DC in the middle), *fft_size = N, or *fft_size = 0 when no spectrum is ready, and re-arms the block.
 * The FFT is hand-written (four-step, radix-2 stages in shared memory; no cuFFT).  Float result against the oracle's double-precision
 * definition: within 2e-4 dB on bins less than 40 dB below the strongest line, every bin's amplitude within 2e-6 of the peak
 * amplitude (FFTW's rounding cannot be reproduced either way).
 * fft_size: power of two in [256, 65536]; window_type: gr::fft::window::win_type (0 Hamming, 1 Hann, 2 Blackman, 3 rectangular,
 * 5 Blackman-Harris; out of range -> Hamming as rx_fft.cpp:176-179; Kaiser / Bartlett / flat-top are not built). */
typedef struct qrl_spectrum qrl_spectrum;
int  qrl_spectrum_create(int fft_size, int window_type, int n_streams, long max_samples, int device, qrl_spectrum** out);
int  qrl_spectrum_destroy(qrl_spectrum*);
int  qrl_spectrum_set_stream(qrl_spectrum*, void* cuda_stream);
int  qrl_spectrum_set_enabled(qrl_spectrum*, int enabled);            /* rx_fft_c::set_enabled */
int  qrl_spectrum_set_fft_size(qrl_spectrum*, int fft_size);          /* rx_fft_c::set_fft_size: buffer and ready flag reset */
int  qrl_spectrum_work(qrl_spectrum*, const float* iq, long T, long stride, int on_device);
int  qrl_spectrum_get(qrl_spectrum*, float* dst, long dst_stride, int dst_on_device, unsigned* fft_size);
long qrl_spectrum_launch_count(qrl_spectrum*);

/* ---- layer-1 deframer on the device (SURVEY.md section 8f row 2) -------------------------------------------------
 * Replaces gr_modem::synchronize / findSync / packBytes (/root/reference/src/gr_modem.cpp:1119-1282, 980-994) for a
 * batch of channels; sync words /root/reference/src/layer1framing.h:8-24.  sync_class: 4 = M17 (0x55F7 / 0xFF5D / 32-bit 0x555D555D,
 * gr_modem.cpp:1187-1207; bit_buf_len 46 * 8, rx_frame_length 46), 1 = "1K" modes (0xB5),
 * 2 = narrow modes (0xED89 voice + 24-bit text / proto / video / callsign / end), 3 = wide modes QPSK250K /
 * QPSKVideo / 4FSK100K (IP / video / end).  bit_buf_len / rx_frame_length as gr_modem::toggleRxMode sets them
 * (gr_modem.cpp:203-322), e.g. 64 / 7 for 4FSK-2k, 1517*8 / 1516 for QPSK-250k.  Input: one decoded bit per byte,
 * [n_channels][stride] with a per-channel count -- exactly qrl_rx_port_device(handle, 2, ...).  Output: per channel
 * up to max_frames records of qrl_deframer_record_bytes() bytes { uint32 frame_type (the sync word), uint32 nbytes,
 * payload }, the arguments of gr_modem::processReceivedData.  State (partial frames, shift register, _modem_sync)
 * carries across calls. */
typedef struct qrl_deframer qrl_deframer;
int  qrl_deframer_create(int sync_class, int bit_buf_len, int rx_frame_length, int n_channels, long max_bits, int max_frames,
                         int device, qrl_deframer** out);
int  qrl_deframer_destroy(qrl_deframer*);
int  qrl_deframer_set_stream(qrl_deframer*, void* cuda_stream);
/* bits [n_channels][stride], counts [n_channels]; on_device = 1: both are device pointers (e.g. from qrl_rx_port_device) */
int  qrl_deframer_work(qrl_deframer*, const unsigned char* bits, const int* counts, long stride, int on_device);
int  qrl_deframer_record_bytes(qrl_deframer*);
/* records_host [n_channels][max_frames][record_bytes] (may be NULL), frame_counts_host [n_channels],
 * modem_sync_host [n_channels] (may be NULL); synchronises */
int  qrl_deframer_read(qrl_deframer*, unsigned char* records_host, int* frame_counts_host, int* modem_sync_host);
int  qrl_deframer_out_device(qrl_deframer*, void** records, int** frame_counts);
int  qrl_deframer_sync(qrl_deframer*);
long qrl_deframer_launch_count(qrl_deframer*);
/* two candidate streams per channel (the two gr_deframer_bb outputs of a dual-decoder mode): like gr_modem::demodulate
 * (/root/reference/src/gr_modem.cpp:1066-1085) the LONGER one of a call is deframed, the first on a tie; same stride for both */
int  qrl_deframer_work2(qrl_deframer*, const unsigned char* bits_a, const int* counts_a, const unsigned char* bits_b, const int* counts_b,
                        long stride, int on_device);
/* frames found beyond max_frames since creation, per channel (they are not stored; frame_counts saturates at max_frames) */
int  qrl_deframer_dropped(qrl_deframer*, int* dropped_host);

/* ---- TX framing: gr_modem::frame (/root/reference/src/gr_modem.cpp:904-961) for a batch of channels -----------------------------------
 * payload [n_channels][payload_stride] with per-channel lengths and frame types (the sync words of layer1framing.h:8-24) ->
 * out [n_channels][out_stride] + lengths: [10 x 0xAA for an IP frame when burst_ip] + sync word (voice: 0xB5 when one_k_mode, else 0xED89
 * + reserved 0xAA; text / video / IP / proto: 24-bit word; other types: none) + payload -- the bytes qrl_tx_work takes.  on_device = 1:
 * all pointers are device pointers, the call is asynchronous on cuda_stream; 0: host pointers, synchronous. */
int  qrl_frame_build(int n_channels, const unsigned char* payload, long payload_stride, const int* payload_len, const unsigned* frame_type,
                     int one_k_mode, int burst_ip, unsigned char* out, long out_stride, int* out_len, int on_device, int device, void* cuda_stream);

/* ---- gr_deframer_bb on the device (/root/reference/src/gr/gr_deframer_bb.cpp:83-185) --------------------------------------------
 * The bit deframer behind ports 2 / 3 of the dual-decoder modes (BPSK, 2FSK, GMSK: gr_demod_base wires _deframer1/2 = type 1,
 * _deframer_700_1/2 = type 2, _deframer_10k_1/2 = type 3).  Input as qrl_deframer_work: one bit per byte, [n_channels][stride] with
 * per-channel counts -- exactly qrl_rx_port_device(handle, 2 or 3, ...).  Output: the stream get_data() hands to gr_modem: for every
 * sync word found, the word itself MSB first (16 bits, 24 for the End word, 8 for type 2) and the next 64 / 32 / 384 input bits;
 * [n_channels][out_stride] with per-channel counts, valid until the next call; feed it to qrl_deframer_work(2) on the device. */
typedef struct qrl_dfbb qrl_dfbb;
int  qrl_dfbb_create(int modem_type /* 1, 2, 3 */, int n_channels, long max_bits, int device, qrl_dfbb** out);
int  qrl_dfbb_destroy(qrl_dfbb*);
int  qrl_dfbb_set_stream(qrl_dfbb*, void* cuda_stream);
int  qrl_dfbb_work(qrl_dfbb*, const unsigned char* bits, const int* counts, long stride, int on_device);
int  qrl_dfbb_out_device(qrl_dfbb*, void** bits, long* stride, int** counts);
int  qrl_dfbb_read(qrl_dfbb*, unsigned char* out_host /* [n_channels][cap] */, long cap, int* counts_host);
int  qrl_dfbb_sync(qrl_dfbb*);
long qrl_dfbb_launch_count(qrl_dfbb*);

/* ---- M17 frame codec on the device (qradiolink_b200/csrc/qrl_m17.cu) --------------------------------------------------------------
 * Receive: M17FrameDecoder (/root/reference/src/M17/M17/M17FrameDecoder.cpp) and the lines of gr_modem::processReceivedData that drive
 * it (/root/reference/src/gr_modem.cpp:1370-1440) for a batch of channels.  Input: the records of the layer-1 deframer (sync class 4),
 * [n_channels][max_frames][record_bytes] of { uint32 frame_type, uint32 nbytes, 46 payload bytes } with per-channel frame_counts --
 * exactly qrl_deframer_out_device(), record_bytes = qrl_deframer_record_bytes() -- or host arrays of the same layout (on_device = 0).
 * max_frames (of the input layout) may not exceed the handle's.  Output, per input record in order, one 56-byte record
 * { uint32 frame_type, lsf[30] (getLsf()), lsf_valid (lsf.valid()), 0, stream_frame[18] (getStreamFrame(): frame number, 16-byte
 * codec2 payload), 0, 0 } as it stands after the record: LSF records (0x55F7) overwrite the LSF whatever its CRC; stream records
 * (0xFF5D) add their LICH segment (a reassembled LSF replaces the current one only if its CRC holds) and decode the stream frame; an
 * EOT record (0x555D555D) reports the current LSF, then resets the channel's decoder if that LSF is valid; other types change nothing.
 * State (LSF, partial LSF, segment map, stream frame) carries across calls.  Records are valid until the next work call. */
typedef struct qrl_m17_rx qrl_m17_rx;
int  qrl_m17_rx_create(int n_channels, int max_frames, int device, qrl_m17_rx** out);
int  qrl_m17_rx_destroy(qrl_m17_rx*);
int  qrl_m17_rx_set_stream(qrl_m17_rx*, void* cuda_stream);
int  qrl_m17_rx_work(qrl_m17_rx*, const unsigned char* records, const int* frame_counts, int record_bytes, int max_frames, int on_device);
/* M17FrameDecoder::reset for one channel */
int  qrl_m17_rx_reset(qrl_m17_rx*, int channel);
/* records_host [n_channels][max_frames][56] (may be NULL), counts_host [n_channels]; synchronises */
int  qrl_m17_rx_read(qrl_m17_rx*, unsigned char* records_host, int* counts_host);
int  qrl_m17_rx_out_device(qrl_m17_rx*, void** records, int** counts);
int  qrl_m17_rx_sync(qrl_m17_rx*);
long qrl_m17_rx_launch_count(qrl_m17_rx*);
/* Transmit: M17Transmitter::start / send (/root/reference/src/M17/M17/M17Transmitter.cpp) and gr_modem::endTransmission's M17 tail
 * (gr_modem.cpp:680-735, 719-728, 868-882) for a batch of channels.  set_lsf: the 28 LSF bytes before the CRC (dst, src, type, meta; a
 * C++ caller fills them with M17LinkSetupFrame); the handle adds the CRC and the six Golay-coded LICH segments.  work: ops [n_channels][K]
 * and payloads [n_channels][K][16], K <= max_steps; op 0 = none, 1 = start (counters reset; 48 x 0x77 preamble, then the LSF frame:
 * 96 bytes), 2 = stream frame (48 bytes), 3 = last stream frame, then 8 x 0x55 0x5D (64 bytes); other values count as none.  Output:
 * [n_channels][stride = max_steps * 96] bytes with per-channel counts, valid until the next work call -- with the same ops on every
 * channel, the input of qrl_tx_work(QRL_MOD_M17, ..., on_device = 1) as it is.  Frame number ((fn + 1) & 0x7FF) and LICH index (mod 6)
 * carry across calls. */
typedef struct qrl_m17_tx qrl_m17_tx;
int  qrl_m17_tx_create(int n_channels, int max_steps, int device, qrl_m17_tx** out);
int  qrl_m17_tx_destroy(qrl_m17_tx*);
int  qrl_m17_tx_set_stream(qrl_m17_tx*, void* cuda_stream);
int  qrl_m17_tx_set_lsf(qrl_m17_tx*, int channel, const unsigned char* lsf28);
int  qrl_m17_tx_work(qrl_m17_tx*, const unsigned char* ops, const unsigned char* payloads, int K, int on_device);
/* out_host [n_channels][cap] (may be NULL), counts_host [n_channels]; synchronises */
int  qrl_m17_tx_read(qrl_m17_tx*, unsigned char* out_host, long cap, int* counts_host);
int  qrl_m17_tx_out_device(qrl_m17_tx*, void** out, long* stride, int** counts);
int  qrl_m17_tx_sync(qrl_m17_tx*);
long qrl_m17_tx_launch_count(qrl_m17_tx*);

/* ---- DMR burst decoder (qrl_dmr.cu): gr_dmr_sink's burst search and the per-burst work of DMRFrame (constructor, setDownlink,
 * validate), CDMREMB::putData and, when ambe_fec is set, CAMBEFEC::regenerateDMR (/root/reference/src/gr/gr_dmr_sink.cpp,
 * src/DMR/dmrframe.cpp, src/DMR/dmrcontrol.cpp:225-271) for a batch of channels.  Input: QRL_DEMOD_DMR's port 2, one hard bit per byte,
 * [n_channels][stride] with per-channel counts (count <= max_bits) -- exactly qrl_rx_port_device(handle, 2, ...) -- or host arrays of
 * the same layout (on_device = 0).  With on_device = 1 the caller guarantees 0 <= counts[c] <= stride (port 2 does); host input is
 * checked, and stride may not exceed max_bits there.  Output, per channel in the order of gr_dmr_sink's _frame_buffer, up to max_bursts records of
 * QRL_DMR_RECORD_BYTES (72) bytes:
 *    0 int64  position: stream index of the burst's last bit, counted from create / reset
 *    8 u8     ts_index (the sink buffer the burst was cut from), 9 frame_type (0 data, 1 voice, 2 voice sync), 10 FN (setFN),
 *   11 u8     downlink, 12 cach_decoded, 13 AT, 14 slot number, 15 LCSS (setDownlink)
 *   16 u8     colour code (255 for voice bursts), 17 data type (DT_VOICE 0xF1 / DT_VOICE_SYNC 0xF0 for voice bursts)
 *   18 u8     validate(), 19 FLCO, 20 FID, 21 EMB colour code, 22 EMB PI, 23 EMB LCSS (voice bursts B-F; 0 otherwise)
 *   24 u32    src ID, 28 u32 dst ID (as validate() leaves them)
 *   32 int32  AMBE error count of regenerateDMR (-1: ambe_fec off or not a voice burst)
 *   36 u8[3]  CACH bytes, 39 u8[33] burst bytes, as the reference leaves them (data bursts re-encoded by a successful validate(),
 *             voice bursts regenerated by the AMBE FEC when it is on)
 * Bursts beyond max_bursts advance the state but are not stored (qrl_dmr_rx_dropped counts them); the DMRTiming calls the reference
 * makes for them (set_slot_times) cannot be replayed, so size max_bursts for a call's worst case (one burst per 288 bits).  Sink state carries across calls;
 * records are valid until the next work call. */
#define QRL_DMR_RECORD_BYTES 72
typedef struct qrl_dmr_rx qrl_dmr_rx;
int  qrl_dmr_rx_create(int n_channels, long max_bits, int max_bursts, int ambe_fec, int device, qrl_dmr_rx** out);
int  qrl_dmr_rx_destroy(qrl_dmr_rx*);
int  qrl_dmr_rx_set_stream(qrl_dmr_rx*, void* cuda_stream);
int  qrl_dmr_rx_work(qrl_dmr_rx*, const unsigned char* bits, const int* counts, long stride, int on_device);
int  qrl_dmr_rx_record_bytes(qrl_dmr_rx*);
/* records_host [n_channels][max_bursts][72] (may be NULL), counts_host [n_channels]; synchronises */
int  qrl_dmr_rx_read(qrl_dmr_rx*, unsigned char* records_host, int* counts_host);
int  qrl_dmr_rx_out_device(qrl_dmr_rx*, void** records, int** counts);
/* bursts not stored because a call found more than max_bursts, per channel, since create / that channel's reset; synchronises */
int  qrl_dmr_rx_dropped(qrl_dmr_rx*, int* dropped_host);
/* gr_dmr_sink's constructor state for one channel (-1 = all): slots idle, buffers empty, position 0 */
int  qrl_dmr_rx_reset(qrl_dmr_rx*, int channel);
int  qrl_dmr_rx_sync(qrl_dmr_rx*);
long qrl_dmr_rx_launch_count(qrl_dmr_rx*);

/* ---- DMR direct-mode (DMO) burst decoder (qrl_dmr.cu): gr_dmr_dmo_sink (the reference's src/gr/gr_dmr_dmo_sink.cpp, after MMDVM's
 * DMRDMORX) and then the per-burst work of qrl_dmr_rx, for a batch of channels.  This is what gr_modem reads when Settings::dmr_mode is
 * DMR_MODE_DMO (radio to radio, no repeater).  Input: QRL_DEMOD_DMR's port 3, the RRC symbol filter's float output at 24 ksps,
 * 5 samples per symbol: [n_channels][stride] floats, channel c takes counts[c] samples (counts == NULL: every channel takes n, which is
 * port 3's case: it has port 0's count on every channel and qrl_rx_port_device returns no count array for it).  0 <= n <= max_samples,
 * stride >= n; on_device = 1: samples (and counts, if given) are device pointers and the caller guarantees 0 <= counts[c] <= n (the
 * kernel clamps to that range); host counts are checked.
 * The sink runs per sample: a 1440-sample ring, the MS data / voice sync searched at every sample while idle (at most 2 of the 24 sign
 * bits wrong, then at most 3 of the 48 sliced sync bits wrong, accepted only above the best correlation so far), then only at the
 * accepted sync's sample +-1; 269 samples after the sync, 132 symbols are sliced with the average of the last four centres and
 * thresholds, and the state machine on the sync kind writes a frame or not.  BS syncs are never matched.  As in the reference, the
 * slice starts 654 samples before the end pointer, so its last symbol comes from the ring slot after the end pointer, which holds the
 * sample from 1439 samples earlier: the last dibit of byte 32 is not the burst's.  Every float operation
 * rounds as the reference's separate SSE multiplies and adds do, in its order; NaN, -0 and denormal samples behave as on the host.
 * Where the reference is undefined the handle defines: the ring, the five sign registers, the four centres and thresholds and the
 * sync kind are zero at create and reset (the reference's constructor leaves them uninitialised).
 * Output, per channel in the order gr_dmr_dmo_sink::writeFrame pushes them, up to max_bursts records of QRL_DMR_RECORD_BYTES in
 * qrl_dmr_rx's layout, with these DMO values:
 *    position: stream index of the sample whose processing wrote the frame, counted from create / reset
 *    ts_index 0, downlink 0, cach_decoded 0, AT 0, LCSS 0, CACH bytes 0 (DMRFrame's defaults; the sink calls setDownlink(false))
 *    slot number 2 and colour code the sink's m_colorCode (writeFrame's setSlotNo(2), setColorCode: on every frame, voice included;
 *    0 after a reset); FN the sink's m_n (0 for syncs and headers, cycling 1..5, 0 for voice bursts without sync)
 *    data type from DMRFrame's constructor (its CDMRSlotType for data frames, DT_VOICE / DT_VOICE_SYNC otherwise); validate(), IDs,
 *    EMB, AMBE error count and burst bytes as qrl_dmr_rx.
 * Bursts beyond max_bursts advance the state but are not stored (qrl_dmr_dmo_rx_dropped counts them).  A burst can follow 270
 * samples after a reset, so max_bursts = max_samples / 270 + 2 never drops.  State carries across calls; records are valid until the
 * next work call. */
typedef struct qrl_dmr_dmo_rx qrl_dmr_dmo_rx;
int  qrl_dmr_dmo_rx_create(int n_channels, long max_samples, int max_bursts, int ambe_fec, int device, qrl_dmr_dmo_rx** out);
int  qrl_dmr_dmo_rx_destroy(qrl_dmr_dmo_rx*);
int  qrl_dmr_dmo_rx_set_stream(qrl_dmr_dmo_rx*, void* cuda_stream);
int  qrl_dmr_dmo_rx_work(qrl_dmr_dmo_rx*, const float* samples, long n, const int* counts, long stride, int on_device);
int  qrl_dmr_dmo_rx_record_bytes(qrl_dmr_dmo_rx*);
/* records_host [n_channels][max_bursts][72] (may be NULL), counts_host [n_channels]; synchronises */
int  qrl_dmr_dmo_rx_read(qrl_dmr_dmo_rx*, unsigned char* records_host, int* counts_host);
int  qrl_dmr_dmo_rx_out_device(qrl_dmr_dmo_rx*, void** records, int** counts);
/* bursts not stored because a call found more than max_bursts, per channel, since create / that channel's reset; synchronises */
int  qrl_dmr_dmo_rx_dropped(qrl_dmr_dmo_rx*, int* dropped_host);
/* gr_dmr_dmo_sink's constructor state for one channel (-1 = all), with ring, registers and position zero.  This is not the sink's own
 * partial reset(), which the state machine runs after a CSBK, a terminator or 13 bursts without sync */
int  qrl_dmr_dmo_rx_reset(qrl_dmr_dmo_rx*, int channel);
int  qrl_dmr_dmo_rx_sync(qrl_dmr_dmo_rx*);
long qrl_dmr_dmo_rx_launch_count(qrl_dmr_dmo_rx*);

/* ---- DMR burst encoder (qrl_dmr.cu): DMRControl's transmit side (/root/reference/src/DMR/dmrcontrol.cpp:19-223) as gr_modem drives
 * it (src/gr_modem.cpp:676-678 startTransmission's CSBK, 710-717 endTransmission, 747-764 transmitDMRHeader, 766-802 transmitDMR),
 * the burst encoders behind DMRFrame (src/DMR/dmrframe.cpp:20-34, 88-96, 399-421, 460-501) and gr_dmr_source's framing
 * (src/gr/gr_dmr_source.cpp:58-126), for a batch of channels.
 * Settings (qrl_dmr_tx_set_config, channel -1 = all; QRL_EINVAL for a value out of range): colour code 0-15, timeslot 1 or 2, 24-bit
 * source and destination IDs, private_call (0: FLCO_GROUP, 1: FLCO_USER_USER, from dmr_call_type), codec2 (FID 0xC2 on the voice LC:
 * !Settings::dmr_vocoder, dmrcontrol.cpp:29-31, 85-86) and up to 27 talker-alias bytes (the UTF-8 prefix DMRControl copies into _ta_tx,
 * dmrcontrol.cpp:33-35, 49-51; zero padded).  They take effect where the reference reads them: every CSBK, header and terminator op
 * reads colour code, slot, IDs and call type, every voice burst colour code and slot (dmrcontrol.cpp:87-89, 104-110, 122-127, 147-148);
 * the header op snapshots the voice LC, _FLCO_TX and the embedded LC (getVoiceHeader, :80-86) and the talker alias (initVoiceTX,
 * :44-52); create and reset snapshot all of them (the constructor, :19-36).  qrl_dmr_tx_create starts every channel in the constructor
 * state of the default config (colour code 1, slot 1, source 1, destination 9, group call, codec2 = 1, no alias: settings.cpp:85-94);
 * qrl_dmr_tx_reset(channel, -1 = all) puts a channel into the constructor state of the config in force, byte position 0.
 * Work: ops [n_channels][K] and audio [n_channels][K][9] (one 9-byte vocoder frame per op), K <= max_ops (QRL_ERANGE otherwise); host
 * arrays, or device arrays with on_device = 1.  One op is one call of the reference:
 *   0 none (so is any value above 4);
 *   1 CSBK: getStartCSBK, 3 CSBK bursts (CSBKO_BSDWNACT with LB set, CBF 0, data1 0, src, dst; CRC-CCITT ^ 0xA5A5, BPTC(196,96));
 *   2 voice header: getVoiceHeader, 2 LC header bursts (RS(12,9) ^ 0x969696, BPTC), then initVoiceTX (FN 0, superframe 0, active);
 *   3 audio: transmitDMR with the op's vocoder frame.  Dropped while idle.  Otherwise the frame joins the pending ones; at three,
 *     getTxAudio makes either one voice burst (FN 0: voice sync; FN 1-5: EMB + embedded-LC fragment) or, when ending at FN 0, the
 *     terminator, the terminator again and two empty frames; FN runs 0-5, the superframe 0-4, superframes 1-4 carry the talker-alias LCs;
 *   4 stop: stopVoiceTX, no burst; it sets the ending state even from idle, as the reference does.
 * Output, valid until the next work call: bytes [n_channels][stride = max_ops * 4 * 72], every burst its 33 frame bytes then 39 zero
 * bytes as gr_dmr_source::set_data appends them, counts in bytes -- with equal counts on every channel, the input of
 * qrl_tx_work(QRL_MOD_DMR, ..., on_device = 1) as it stands; and per channel up to max_ops * 4 records of QRL_DMR_TX_RECORD_BYTES (16):
 *    0 int64  position of the burst's first byte in the channel's byte stream since create / reset
 *    8 u8     slot number the frame carries (the configured slot; 0 for the two empty frames): gr_dmr_source's get_slot_times argument
 *    9 u8     kind: 1 CSBK, 2 LC header, 3 voice sync (FN 0), 4 voice (FN 1-5), 5 terminator with LC, 6 empty
 *   10 u8     FN, 11 u8 LCSS of the embedded fragment (FN 1: 1, FN 2-3: 3, FN 4: 2, otherwise 0)
 *   12 int32  index of the op (within the call) that produced the burst
 * An adapter attaches gr_dmr_source's tags from a record: tx_time on byte `position` (DMRTiming::get_slot_times(slot) on the host) and
 * zero_samples on byte position + 33 with 780 samples (qrl_tx_zero_samples).  All syncs are the MS-sourced words (duplex = false).
 * Where the reference is undefined or accidental, this is the definition:
 *   - DMRFrame(uint8_t) leaves _data_type uninitialised, so transmitDMR's DT_TERMINATOR_WITH_LC test reads garbage for a voice frame:
 *     here a voice burst is never a terminator;
 *   - the two empty frames are 33 zero bytes with slot 0;
 *   - the terminator is a fresh CDMRLC(_FLCO_TX, src, dst): FID 0 even for codec2 (getVoiceTerminator, :120-128);
 *   - FN 5 carries CDMREmbeddedData::getData's null fragment, LCSS 0;
 *   - up to two pending vocoder frames carry across calls; a terminator drops them (clearTxAudio), a new header does not.
 * State (counters, snapshots, pending frames, byte position) carries across calls. */
#define QRL_DMR_TX_RECORD_BYTES 16
typedef struct qrl_dmr_tx_config {
    int color_code;                  /* 0-15 */
    int timeslot;                    /* 1 or 2 */
    unsigned src_id, dst_id;         /* 24 bit */
    int private_call;                /* 0: FLCO_GROUP, 1: FLCO_USER_USER */
    int codec2;                      /* 1: FID 0xC2 on the voice LC (Settings::dmr_vocoder == 0) */
    int talker_alias_len;            /* 0-27 */
    unsigned char talker_alias[28];  /* the first talker_alias_len bytes are used */
} qrl_dmr_tx_config;
typedef struct qrl_dmr_tx qrl_dmr_tx;
int  qrl_dmr_tx_create(int n_channels, int max_ops, int device, qrl_dmr_tx** out);
int  qrl_dmr_tx_destroy(qrl_dmr_tx*);
int  qrl_dmr_tx_set_stream(qrl_dmr_tx*, void* cuda_stream);
int  qrl_dmr_tx_set_config(qrl_dmr_tx*, int channel, const qrl_dmr_tx_config* cfg);
int  qrl_dmr_tx_reset(qrl_dmr_tx*, int channel);
int  qrl_dmr_tx_work(qrl_dmr_tx*, const unsigned char* ops, const unsigned char* audio, int K, int on_device);
/* bytes_host [n_channels][cap] (may be NULL), records_host [n_channels][max_ops * 4][16] (may be NULL), counts_host [n_channels]
 * (bytes; records = counts / 72); synchronises */
int  qrl_dmr_tx_read(qrl_dmr_tx*, unsigned char* bytes_host, long cap, unsigned char* records_host, int* counts_host);
int  qrl_dmr_tx_out_device(qrl_dmr_tx*, void** bytes, long* stride, int** counts, void** records);
int  qrl_dmr_tx_sync(qrl_dmr_tx*);
long qrl_dmr_tx_launch_count(qrl_dmr_tx*);

/* ---- stand-alone kernels exposed for tests / micro-benchmarks ---- */
/* batched decimating FIR (stage 1 alone): x [C][T] device, y [C][ceil(T/D)] device; zero history */
int qrl_fir_decim_ccf_device(const float* taps, int ntaps, int D, const float* x_dev, long T, long x_stride,
                             float* y_dev, long y_stride, int C, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif
