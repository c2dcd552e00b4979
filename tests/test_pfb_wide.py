"""CPU tier: the polyphase channelizer / synthesizer past 64 channels through the library's own sources run on host threads
(tools/emu/build_emulated_lib.py): pfb_fir_kernel + pfb_dft_kernel bit-identical to the oracle at M = 65, 100, 256 with 1, 2, 34 and
128 taps per branch, in ragged chunks, host input and device input 8 bytes past a boundary; the M = 4096 limit of create."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_pfb(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, _ = build(str(tmp_path_factory.mktemp("qrl_emu_pfb")))
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    yield q
    L._LIB_PATH, L._LIB = saved


def _host_as_device(x):
    """the emulated library's device memory is host memory: a host array 8 bytes past a 16-byte boundary stands for a device pointer"""
    buf = np.zeros(x.size + 2, np.complex64)
    k = 1 if buf.ctypes.data % 16 == 0 else 0
    buf[k:k + x.size] = np.ascontiguousarray(x).reshape(-1)
    ptr = buf.ctypes.data + 8 * k
    assert ptr % 16 == 8
    return ptr, buf


@pytest.mark.parametrize("tpf", [1, 2, 34, 128])
@pytest.mark.parametrize("M", [65, 100, 256])
def test_wide_channelizer_emulated(emu_pfb, oracle, M, tpf):
    from tests import test_gpu_pfb_wide as TG
    # 1, M - 3, not multiples of M, more than one CTA tile of either kernel (72 FIR / 64 DFT output times)
    sizes = [1, M - 3, 75 * M + 11, 2 * M - 1]
    TG.chan_parity(emu_pfb, oracle, M, TG.rand_taps(M, tpf * M - (M // 3 if tpf > 1 else 0)), sizes, ("host", "dev"), _host_as_device)


@pytest.mark.parametrize("tpf", [1, 2, 34, 128])
@pytest.mark.parametrize("M", [65, 100, 256])
def test_wide_synthesizer_emulated(emu_pfb, oracle, M, tpf):
    from tests import test_gpu_pfb_wide as TG
    TG.synth_parity(emu_pfb, oracle, M, TG.rand_taps(M + 1, tpf * M - (M // 5 if tpf > 1 else 0)), [1, 70, 3, 9], ("dev", "host"),
                    _host_as_device)


def test_create_limits_emulated(emu_pfb):
    """4096 channels of 25 kHz (102.4 Msps) is the widest bank: M = 4097 fails at create with the limit named"""
    emu_pfb.PfbChannelizer(4096, np.ones(4096 * 128, np.float32), max_in=8192).close()
    emu_pfb.PfbSynthesizer(4096, np.ones(4096, np.float32), max_in=4).close()
    for cls in (emu_pfb.PfbChannelizer, emu_pfb.PfbSynthesizer):
        with pytest.raises(emu_pfb.QrlError, match="M above 4096"):
            cls(4097, np.ones(4097, np.float32), max_in=16)
    with pytest.raises(emu_pfb.QrlError, match="bad argument"):
        emu_pfb.PfbChannelizer(256, np.ones(256 * 128 + 1, np.float32), max_in=16)
