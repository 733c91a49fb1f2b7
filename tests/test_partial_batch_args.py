"""Session sizes outside 1..batch are refused before anything touches a device."""
import pytest

import smaat_unet_b200 as S
from smaat_unet_b200.engine import InferenceSession
from smaat_unet_b200.train import TrainSession


@pytest.mark.parametrize("sizes", [(0,), (9,), (3, 9), (-1,)])
@pytest.mark.parametrize("cls", [InferenceSession, TrainSession])
def test_batch_sizes_outside_the_capacity_raise(cls, sizes):
    with pytest.raises(ValueError, match="batch_sizes"):
        cls(S.SmaAt_UNet(12, 1), 8, (12, 32, 32), batch_sizes=sizes)
