"""CPU tier: the FreeDV chains of the library's own sources on host threads (tools/emu/build_emulated_lib.py, see
tests/test_emulated_library.py) -- handle creation, stage-1 / side-band / AGC / int16 kernels, the feedforward AGC and the x125
interpolator -- against the committed known answers, bit for bit, and the QRL_EINVAL paths of the two factories."""
import pytest

from tests import test_freedv as TF
from tests.golden import freedv_cases as F
from tests.test_emulated_library import emu_qrl  # noqa: F401  (module-scoped fixture: the emulated build)

pytestmark = pytest.mark.timeout(900)


@pytest.mark.parametrize("name", sorted(F.RX_CASES))
def test_freedv_rx_golden_through_the_emulated_library(emu_qrl, name):  # noqa: F811
    TF.golden_rx_through(emu_qrl, name)


@pytest.mark.parametrize("name", sorted(F.TX_CASES))
def test_freedv_tx_golden_through_the_emulated_library(emu_qrl, name):  # noqa: F811
    TF.golden_tx_through(emu_qrl, name)


def test_freedv_einval_through_the_emulated_library(emu_qrl):  # noqa: F811
    TF.einval_paths(emu_qrl)
