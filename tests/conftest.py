import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _make(directory, *targets):
    subprocess.run(["make", "-C", directory, *targets], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)


@pytest.fixture(scope="session")
def emu_lib():
    """Test-only CPU emulation build of the product sources (tests/emu)."""
    from sunscreen_b200.lib import B200Lib
    _make(os.path.join(ROOT, "tests", "emu"))
    return B200Lib(os.path.join(ROOT, "tests", "emu", "_build", "libb200bfv_emu.so"), _allow_emu=True)


@pytest.fixture(scope="session")
def port():
    """The plain-C restatement of the path (oracle/bfv_oracle.c)."""
    import oracle_port
    _make(os.path.join(ROOT, "oracle"), "port")
    return oracle_port.OraclePort()


@pytest.fixture(scope="session")
def ref():
    """The unmodified reference (oracle/_ref/libsealc_ref.so), as build() compiles it where the reference sources exist."""
    import refseal
    if not refseal.have_ref():
        pytest.skip("reference library oracle/_ref/libsealc_ref.so not available")
    return refseal.RefLib.get()
