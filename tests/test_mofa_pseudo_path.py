"""CPU: which path (dense pseudo-data or sparse) a poisson / bernoulli MOFA view takes."""
import pytest

from muon_b200._mofa import _pseudo_path

GB = 1 << 30


@pytest.mark.parametrize("sparse_input", [True, False])
def test_auto_keeps_dense_whenever_it_fits(sparse_input):
    # 12 B per element against 60 % of the free memory
    assert _pseudo_path(sparse_input, (400, 70), 10 * GB, "auto") == "dense"
    assert _pseudo_path(sparse_input, (100_000, 42_949), 80 * GB, "auto") == "dense"      # just under 48 GiB


def test_auto_takes_sparse_only_for_sparse_inputs_that_do_not_fit():
    assert _pseudo_path(True, (100_000, 200_000), 80 * GB, "auto") == "sparse"
    assert _pseudo_path(True, (100_000, 42_950), 80 * GB, "auto") == "sparse"            # just over 48 GiB
    # a dense array that does not fit keeps the dense path (which refuses it)
    assert _pseudo_path(False, (100_000, 200_000), 80 * GB, "auto") == "dense"


@pytest.mark.parametrize("sparse_input", [True, False])
@pytest.mark.parametrize("shape", [(10, 10), (500_000, 200_000)])
def test_forced_paths(sparse_input, shape):
    assert _pseudo_path(sparse_input, shape, 80 * GB, "dense") == "dense"
    assert _pseudo_path(sparse_input, shape, 80 * GB, "sparse") == "sparse"


def test_unknown_mode_is_an_error():
    with pytest.raises(ValueError):
        _pseudo_path(True, (10, 10), GB, "Sparse")
