"""CPU: the Optimizer takes GBRT only as a GbrtEngine instance; the string and any other object are refused before a device is
touched."""
import pytest

from kubeflow_b200.optimizer import Optimizer
from kubeflow_b200.space import Real


@pytest.mark.parametrize("est", ["GBRT", "gbrt", object(), 3])
def test_gbrt_needs_an_engine_instance(est):
    with pytest.raises(ValueError, match="GbrtEngine"):
        Optimizer([Real(0.0, 1.0)], base_estimator=est)
