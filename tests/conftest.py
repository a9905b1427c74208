import os, sys, pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


ORACLE_SO = os.path.join(ROOT, "oracle", "_build", "libkj_oracle.so")
EMU_SO = os.path.join(ROOT, "tests", "emu", "_build", "libkjb_emu.so")
CUDA_SO = os.path.join(ROOT, "kajiya_b200", "csrc", "libkjb.so")


def _ensure_built(path, target):
    if not os.path.exists(path):
        import __graft_entry__ as g
        getattr(g, target)()
    return path


@pytest.fixture(scope="session")
def oracle_lib():
    from kajiya_b200._abi import KjbLib
    return KjbLib(_ensure_built(ORACLE_SO, "build_oracle"))


@pytest.fixture(scope="session")
def emu_lib():
    from kajiya_b200._abi import KjbLib
    return KjbLib(_ensure_built(EMU_SO, "build_emu"))


@pytest.fixture(scope="session")
def cuda_lib():
    import kajiya_b200
    return kajiya_b200.lib()   # raises if the extension is missing: GPU tests must never fall back
