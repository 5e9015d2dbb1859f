"""GPU: the training step (Phenaki.forward -> phk_maskgit_train_step: forward, loss and the hand-written backward
kernels of csrc/train.cu) against the reference's autograd loss and gradients (tests/golden/train_*.pt): fp32 mode at
parity tolerances, bf16 mode (wgmma products) within 5 % of each gradient tensor's largest entry."""
import pytest

from tests import cases as C
from tests import gpu_train_check as T

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(C.TRAIN_CASES))
def test_training_step_matches_reference_autograd(name):
    T.check_case(name, verbose=False)


@pytest.mark.parametrize("name", ["generator", "with_critic"])
def test_training_step_bf16_mode_is_close_to_reference_autograd(name):
    T.check_case(name, verbose=False, bf16=True)
