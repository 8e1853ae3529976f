"""The drop-in boundary: libprl.so loads, exports every symbol include/prl.h declares, and the product
package never touches oracle/.  No compute calls here (CPU box)."""
import ast
import ctypes
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def built_lib():
    from pipelinerl_b200 import _build, _lib
    _build.build(verbose=False)
    return _lib.load()


def _header_symbols():
    text = (ROOT / "include" / "prl.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(prl_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol(built_lib):
    from pipelinerl_b200 import _lib
    syms = _header_symbols()
    assert syms, "no symbols parsed from include/prl.h"
    for s in syms:
        assert hasattr(built_lib, s), f"libprl.so does not export {s}"
    assert sorted(_lib.declared_symbols()) == syms, "ctypes binding and header disagree"


def test_version_and_error_string(built_lib):
    assert built_lib.prl_version() >= 100
    assert isinstance(built_lib.prl_last_error(), bytes)
    assert built_lib.prl_pg_workspace_bytes(16) > 0 and built_lib.prl_adamw_workspace_bytes() > 0


def test_sm90a_cubin_present():
    import subprocess
    from pipelinerl_b200 import _lib
    out = subprocess.run(["cuobjdump", "--list-elf", str(_lib.lib_path())], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out


def test_product_never_imports_oracle():
    for py in (ROOT / "pipelinerl_b200").rglob("*.py"):
        tree = ast.parse(py.read_text())
        for node in ast.walk(tree):
            names = []
            if isinstance(node, ast.Import):
                names = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom) and node.module:
                names = [node.module]
            assert not any(n == "oracle" or n.startswith("oracle.") for n in names), f"{py} imports oracle"


def test_ops_fail_loudly_without_cuda():
    import torch
    from pipelinerl_b200.finetune.optim import FusedAdamW
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    p = torch.nn.Parameter(torch.zeros(4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        FusedAdamW([("w", p)], lr=1e-3)


def test_argument_validation_needs_no_gpu(built_lib):
    """Every entry point validates its arguments BEFORE touching CUDA: bad shapes come back as a negative status with a
    message (the C ABI never throws).  Dummy non-NULL pointers are never dereferenced on these paths."""
    lib, P = built_lib, 0x1000
    cases = [
        (lambda: lib.prl_gemm_ex(P, 20, 0, P, 24, 0, 16, 16, 20, P, 16, 0, 0, None, None, 0, 1.0, None), b"multiples of 8"),
        (lambda: lib.prl_gemm_ex(P, 24, 0, P, 24, 0, 16, 16, 24, P, 16, 0, 1, None, None, 0, 1.0, None), b"accumulate"),
        (lambda: lib.prl_gemm_ex(P, 24, 0, P, 24, 0, 16, 16, 24, P, 8, 0, 0, None, None, 0, 1.0, None), b"ldc"),
        (lambda: lib.prl_gemm_ex(None, 8, 0, P, 8, 0, 8, 8, 8, P, 8, 0, 0, None, None, 0, 1.0, None), b"NULL"),
        (lambda: lib.prl_transpose_bf16(P, 8, 16, 8, P, 8, None), b"bad shape"),
        (lambda: lib.prl_rmsnorm_fwd(P, P, 4, 12, 1e-6, P, P, None), b"multiple of 8"),
        (lambda: lib.prl_rmsnorm_fwd(P, P, 4, 16384, 1e-6, P, P, None), b"8192"),
        (lambda: lib.prl_rope_inplace(P, 256, 4, 2, 100, P, P, 1.0, None), b"head_dim"),
        (lambda: lib.prl_silu_mul_fwd(P, 4, 12, P, None), b"I % 8"),
        (lambda: lib.prl_paged_attn_prefill_tc(P, 8, P, 4, 1, 0, P, 4, P, P, P, P, 1, 8, 4, 2, 64, 64, 0.1, P, None),
         b"head_dim"),
        (lambda: lib.prl_paged_attn_prefill_tc(P, 8, P, 4, 1, 3, P, 4, P, P, P, P, 1, 8, 4, 2, 128, 64, 0.1, P, None),
         b"bad layer"),
        (lambda: lib.prl_head_logprob(P, None, P, 4, 16, 12, 1.0, None, 1, 0, 0, None, None, None, None, None, P, 1 << 20,
                                      None), b"K % 8"),
    ]
    for call, needle in cases:
        assert call() < 0
        assert needle in lib.prl_last_error(), (needle, lib.prl_last_error())


def test_header_is_plain_c():
    """include/prl.h is the drop-in boundary: it must compile as C99 (plain pointers and sizes, no C++/torch types)."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    for std, lang in (("-std=c99", "c"), ("-std=c++17", "c++")):
        r = subprocess.run(["gcc", std, "-fsyntax-only", "-Wall", "-x", lang, str(ROOT / "include" / "prl.h")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr


def test_plain_c_client_links_and_calls(built_lib, tmp_path):
    """tests/c_abi/client.c — a C program that knows only include/prl.h — links against libprl.so and runs."""
    import os
    import shutil
    import subprocess
    from pipelinerl_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    so = Path(_lib.lib_path())
    exe = tmp_path / "client"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-I", str(ROOT / "include"), str(ROOT / "tests" / "c_abi" / "client.c"),
                        "-L", str(so.parent), "-lprl", f"-Wl,-rpath,{so.parent}", "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    env = dict(os.environ, LD_LIBRARY_PATH=f"{so.parent}:{os.environ.get('LD_LIBRARY_PATH', '')}")
    r = subprocess.run([str(exe)], capture_output=True, text=True, env=env, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("ok version="), (r.returncode, r.stdout, r.stderr)
