"""pytest configuration: registers the `gpu` marker and the shared parity-checker fixtures."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def orc():
    from _oracle import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def ref():
    from _oracle import Ref
    try:
        return Ref()
    except (FileNotFoundError, OSError) as e:  # pragma: no cover
        pytest.skip(f"compiled reference unavailable: {e}")


@pytest.fixture(scope="session")
def orc10():
    from _oracle import Oracle
    return Oracle(10)


@pytest.fixture(scope="session")
def ref10():
    from _oracle import Ref
    try:
        return Ref(10)
    except (FileNotFoundError, OSError) as e:  # pragma: no cover
        pytest.skip(f"compiled 10-bit reference unavailable: {e}")


@pytest.fixture(scope="session")
def cuda_lib():
    """The product library through its public Python host layer; fails loudly if missing."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import kvazaar_b200 as kb
    return kb
