"""The reference's four offline test files run UNCHANGED against this package on an H100 (VERDICT r1 item 7e, SURVEY #26).

The files under tests/golden/ref_tests/ are verbatim copies (see the README there).  They import ``vit_prisma`` -- here that resolves to
vit-prisma_b200/vit_prisma -- build host-resident models and feed host tensors; the package stages them on the GPU."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = ["test_hooks.py", "test_cache_hook_names.py", "test_weight_properties.py", os.path.join("models", "test_models.py")]


@pytest.mark.parametrize("name", FILES)
def test_reference_test_file_passes_unchanged(name):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.path.join(ROOT, "vit-prisma_b200") + os.pathsep + env.get("PYTHONPATH", "")
    path = os.path.join(ROOT, "tests", "golden", "ref_tests", name)
    out = subprocess.run([sys.executable, "-m", "pytest", path, "-q", "-x", "-p", "no:cacheprovider", "--rootdir", os.path.dirname(path),
                          "-c", os.devnull], cwd=os.path.dirname(path), env=env, capture_output=True, text=True, timeout=900)
    tail = (out.stdout + out.stderr)[-3000:]
    assert out.returncode == 0, tail
    assert " passed" in out.stdout and " failed" not in out.stdout, tail
