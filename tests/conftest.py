"""pytest wiring.

* ``-m "not gpu"`` (run on a CPU-only box): oracle pinning, host logic driven
  through the CPU stand-in of the extension (``oracle.ext_cpu``), C-ABI export
  checks, gloo data-parallel tests.
* ``-m gpu`` (run on an H100): the parity tests proper - the product's CUDA
  path against the oracle on the same seeded inputs, through the C ABI.
"""

import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
for extra in (ROOT, ROOT / "tiny-llm_b200"):
    if str(extra) not in sys.path:
        sys.path.insert(0, str(extra))

os.environ.setdefault("MASTER_ADDR", "127.0.0.1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture
def cpu_ext(monkeypatch):
    """Route the extension's entry points to the CPU oracle so that HOST logic
    (page pools, block tables, scheduler, model wiring) can be tested without a
    GPU.  Test-only: the product never does this."""
    from extensions_b200 import tiny_llm_ext_b200
    from oracle import ext_cpu

    ext_cpu.install(tiny_llm_ext_b200, monkeypatch)
    return tiny_llm_ext_b200


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
