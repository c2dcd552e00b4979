"""Host-side mirror of the reference's TX operator surface: make_gr_mod_4fsk / make_gr_mod_qpsk
(/root/reference/src/gr/gr_mod_4fsk.h:46-48, gr_mod_qpsk.h) batched over channels.  gr_byte_source
(src/gr/gr_byte_source.cpp:54-106) hands the modulator a byte vector; `work(bytes)` is that hand-off."""
import ctypes as C

import numpy as np

from .lib import KIND, PARAM, Handle, check, load_library


class TxBlock(Handle):
    ABI = "tx"

    def __init__(self, kind, sps, samp_rate, carrier_freq, filter_width, flag=0, n_channels=1,
                 max_items=1 << 12, device=0, low_cutoff=None):
        self._L = load_library()
        self.n_channels, self.max_items = int(n_channels), int(max_items)
        if kind == KIND.MOD_FREEDV:
            self._create(self._L.qrl_tx_create_freedv, sps, samp_rate, carrier_freq, filter_width, int(low_cutoff), int(flag),
                         self.n_channels, self.max_items, device)
        else:
            self._create(self._L.qrl_tx_create, kind, sps, samp_rate, carrier_freq, filter_width, int(flag),
                         self.n_channels, self.max_items, device)

    def zero_samples(self, byte_offset, n_samples, channel=-1):
        """gr_mod_dmr: the "zero_samples" tag on input byte `byte_offset` of `channel` (-1: all), see qrl_tx_zero_samples."""
        check(self._L.qrl_tx_zero_samples(self._h, int(channel), int(byte_offset), int(n_samples)), self._h, "zero_samples")

    def set_filter_width(self, filter_width):
        """gr_mod_nbfm::set_filter_width (gr_mod_nbfm.cpp:78-93), mid-stream."""
        check(self._L.qrl_tx_set_param(self._h, -1, PARAM.FILTER_WIDTH, float(filter_width)), self._h, "set_filter_width")

    def set_ctcss(self, value):
        """gr_mod_nbfm::set_ctcss (gr_mod_nbfm.cpp:101-139): 0 = no tone (audio gain 0.98), f = CTCSS tone at f Hz (gain 0.85, 300 Hz high-pass)."""
        check(self._L.qrl_tx_set_param(self._h, -1, PARAM.CTCSS, float(value)), self._h, "set_ctcss")

    def set_bb_gain(self, value):
        check(self._L.qrl_tx_set_param(self._h, -1, PARAM.BB_GAIN, float(value)), self._h, "set_bb_gain")

    set_stream = Handle._set_stream

    def _work(self, data, dtype):
        """[n_channels, n] items of `dtype` from a host array -> complex64 [n_channels, n_out]."""
        data = np.ascontiguousarray(data, dtype)
        if data.ndim == 1:
            data = data[None, :]
        n = data.shape[1]
        check(self._L.qrl_tx_work(self._h, data.ctypes.data_as(C.c_void_p), n, n, 0), self._h, "qrl_tx_work")
        nout = C.c_long()
        check(self._L.qrl_tx_out_device(self._h, None, None, C.byref(nout)), self._h, "tx_out_device")
        out = np.zeros((self.n_channels, max(1, nout.value)), np.complex64)
        n2 = C.c_long()
        check(self._L.qrl_tx_read(self._h, out.ctypes.data_as(C.c_void_p), max(1, nout.value), C.byref(n2), 0), self._h, "qrl_tx_read")
        return out[:, :n2.value]

    def work(self, data):
        """data: uint8 [n_channels, n] frame bytes -> complex64 [n_channels, n_out] at 1 Msps."""
        return self._work(data, np.uint8)

    def work_audio(self, audio):
        """analog modulators (NBFM / SSB): float32 [n_channels, n] audio at 8 ksps -> complex64 [n_channels, n_out]."""
        return self._work(audio, np.float32)

    def work_modem(self, samples):
        """FreeDV: int16 [n_channels, n] modem samples at 8 ksps (what freedv_tx_ss produces) -> complex64 [n_channels, n x sps]."""
        return self._work(samples, np.int16)

    def work_device(self, dev_ptr, n, stride):
        check(self._L.qrl_tx_work(self._h, C.c_void_p(dev_ptr), n, stride, 1), self._h, "qrl_tx_work")

    sync = Handle._sync
    launches = property(Handle._launches)


def make_gr_mod_4fsk(sps, samp_rate, carrier_freq, filter_width, fm, n_channels=1, **kw):
    return TxBlock(KIND.MOD_4FSK, sps, samp_rate, carrier_freq, filter_width, int(bool(fm)), n_channels, **kw)


def make_gr_mod_qpsk(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    return TxBlock(KIND.MOD_QPSK, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_mod_bpsk(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    """src/gr/gr_mod_bpsk.h (instances gr_mod_base.cpp:168-169)."""
    return TxBlock(KIND.MOD_BPSK, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_mod_2fsk(sps, samp_rate, carrier_freq, filter_width, fm, n_channels=1, **kw):
    """src/gr/gr_mod_2fsk.h (instances gr_mod_base.cpp:155-159)."""
    return TxBlock(KIND.MOD_2FSK, sps, samp_rate, carrier_freq, filter_width, int(bool(fm)), n_channels, **kw)


def make_gr_mod_gmsk(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    """src/gr/gr_mod_gmsk.h (instances gr_mod_base.cpp:160-162: sps 50 / 100 / 10 = GMSK2K / 1K / 10K)."""
    return TxBlock(KIND.MOD_GMSK, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_mod_nbfm(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    """src/gr/gr_mod_nbfm.h (instances gr_mod_base.cpp:171-172); feed with TxBlock.work_audio."""
    return TxBlock(KIND.MOD_NBFM, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_mod_ssb(sps, samp_rate, carrier_freq, filter_width, sb, n_channels=1, **kw):
    """src/gr/gr_mod_ssb.h (instances gr_mod_base.cpp:178-179); feed with TxBlock.work_audio."""
    return TxBlock(KIND.MOD_SSB, sps, samp_rate, carrier_freq, filter_width, int(sb), n_channels, **kw)


def make_gr_mod_m17(sps=125, samp_rate=1000000, carrier_freq=1700, filter_width=9000, n_channels=1, **kw):
    """src/gr/gr_mod_m17.h:43-44 (defaults as there); items: frame bytes, 4 symbols per byte, 125 / 3 output samples per 24 ksps
    sample."""
    return TxBlock(KIND.MOD_M17, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_mod_am(sps=125, samp_rate=1000000, carrier_freq=1700, filter_width=5000, n_channels=1, **kw):
    """src/gr/gr_mod_am.h (instance gr_mod_base.cpp:167: make_gr_mod_am(125, 1e6, 1700, 5000)); feed with TxBlock.work_audio."""
    return TxBlock(KIND.MOD_AM, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_mod_dsss(sps=25, samp_rate=1000000, carrier_freq=1700, filter_width=200, n_channels=1, max_items=8, **kw):
    """src/gr/gr_mod_dsss.h (instance gr_mod_base.cpp:170: make_gr_mod_dsss(25, 1e6, 1700, 200)); items: frame bytes at 1 byte/s: every byte
    becomes 10^6 output samples, hence the small default max_items."""
    return TxBlock(KIND.MOD_DSSS, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, max_items=max_items, **kw)


def make_gr_mod_dmr(sps=125, samp_rate=1000000, carrier_freq=1700, filter_width=5000, n_channels=1, **kw):
    """src/gr/gr_mod_dmr.h:37-38 (defaults as there); items: frame bytes, 4 symbols per byte.  TxBlock.zero_samples is the
    "zero_samples" stream tag gr_dmr_source attaches to the bytes of an idle burst (gr_zero_idle_bursts)."""
    return TxBlock(KIND.MOD_DMR, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_mod_freedv(sps=125, samp_rate=8000, carrier_freq=1700, filter_width=2000, low_cutoff=200, mode=0, sb=0, n_channels=1, **kw):
    """src/gr/gr_mod_freedv.h:39-40 (defaults as there; instances gr_mod_base.cpp:181-203, e.g. (125, 1e6, 1700, 2500, 200, MODE_1600, 0))
    behind codec2's freedv_tx_ss: feed int16 modem samples with TxBlock.work_modem.  `mode` is kept as an attribute for the adapter."""
    blk = TxBlock(KIND.MOD_FREEDV, sps, samp_rate, carrier_freq, filter_width, int(sb), n_channels, low_cutoff=low_cutoff, **kw)
    blk.mode = mode
    return blk
