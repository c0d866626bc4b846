"""CPU: the registry's Python wrapper refuses malformed key buffers before it reaches the library (no GPU needed)."""
import numpy as np
import pytest

from ethereum_consensus_b200 import crypto


@pytest.mark.parametrize("nbytes", [1, 47, 49, 95, 48 * 3 + 7])
def test_append_rejects_partial_keys_before_the_library(nbytes):
    reg = crypto.Registry.__new__(crypto.Registry)   # no load: the check must come before any library call
    reg.n = 5
    for buf in (bytes(nbytes), np.zeros(nbytes, np.uint8)):
        with pytest.raises(ValueError, match="48 bytes each"):
            reg.append(buf)
    assert reg.n == 5
