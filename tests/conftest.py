import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def built():
    import __graft_entry__ as g

    g.build()
    return True


@pytest.fixture(scope="session")
def ctx(built):
    import torch
    from hold_b200 import capi

    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    torch.cuda.set_device(0)
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture()
def isolated(built):
    """Run a test function of this suite in a FRESH interpreter (own CUDA context) — for kernels that had no hardware run
    yet: a device fault there must not poison the CUDA context of the session-wide `ctx` and with it every later test.
    Usage: isolated("tests/test_gpu_x.py", "impl_name") -> raises AssertionError with the child's output on failure."""
    import subprocess
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no GPU")

    def run(module_path, func, timeout=240, env=None):
        code = (
            "import sys, importlib.util, torch\n"
            f"sys.path.insert(0, {ROOT!r})\n"
            f"spec = importlib.util.spec_from_file_location('m', {os.path.join(ROOT, module_path)!r})\n"
            "m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)\n"
            "from hold_b200 import capi\n"
            "torch.cuda.set_device(0)\n"
            "c = capi.Context(0)\n"
            f"getattr(m, {func!r})(c)\n"
            "print('ISOLATED-OK')\n"
        )
        e = dict(os.environ, PYTHONPATH=ROOT)
        e.update(env or {})
        r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=e, capture_output=True, text=True, timeout=timeout)
        assert r.returncode == 0 and "ISOLATED-OK" in r.stdout, (r.stdout[-2000:] + "\n" + r.stderr[-4000:])

    return run
