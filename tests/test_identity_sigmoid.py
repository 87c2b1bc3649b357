"""identity.class_probabilities: the class maps' sigmoid in float64, rounded once to float32 (the definition the device's
multi-class step applies to the logits it samples), against the float32 NumPy sigmoid the host chain used before."""
import numpy as np

from sleap_b200.nn import identity


def test_class_probabilities_within_three_ulp_of_the_float32_sigmoid():
    z = np.concatenate([np.linspace(-40, 40, 400001), np.random.default_rng(3).normal(0, 6, 200000)]).astype(np.float32)
    new = identity.class_probabilities(z)
    assert new.dtype == np.float32
    with np.errstate(over="ignore"):
        old = (np.float32(1) / (np.float32(1) + np.exp(-z, dtype=np.float32))).astype(np.float32)
    ulp = np.abs(new.view(np.int32).astype(np.int64) - old.view(np.int32).astype(np.int64))
    assert ulp.max() <= 3                      # the float32 exp and division of the old form round three times
    assert identity.class_probabilities(np.float32(-1000.0)) == 0 and identity.class_probabilities(np.float32(1000.0)) == 1
