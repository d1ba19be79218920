"""-m gpu: the drop-in boundary.  The reference's OWN parity harness (tests/test-backend-ops.cpp, compiled unmodified into
oracle/_ref by oracle/Makefile) is run against the registered "B200" ggml backend: every op the backend claims through
supports_op is executed on the GPU and compared with the reference CPU backend under the reference's NMSE thresholds
(MUL_MAT 5e-4 :1660, SOFT_MAX 1e-6 :2077, others 1e-7 :320)."""
import os
import re
import subprocess
from pathlib import Path

import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
PLUGIN = ROOT / "prima.cpp_b200" / "libggml-b200.so"
OPS = ["MUL_MAT", "RMS_NORM", "ROPE", "SOFT_MAX", "ADD", "MUL", "CPY", "CONT", "DUP", "GET_ROWS", "SILU", "FLASH_ATTN_EXT"]


def run_tbo(args, timeout=900):
    exe = O.ORACLE / "_ref" / "v3" / "test-backend-ops"
    if not exe.exists() or not PLUGIN.exists():
        pytest.skip("oracle/_ref/v3/test-backend-ops or libggml-b200.so not built (build() builds them only where the reference source tree is readable)")
    env = dict(os.environ, LD_PRELOAD=str(PLUGIN))
    p = subprocess.run([str(exe)] + args, env=env, capture_output=True, text=True, timeout=timeout)
    return p.returncode, re.sub(r"\x1b\[[0-9;]*m", "", p.stdout + p.stderr)


@pytest.mark.parametrize("op", OPS)
def test_reference_test_backend_ops(cuda, op):
    rc, out = run_tbo(["test", "-b", "B200_0", "-o", op])
    tail = "\n".join(out.splitlines()[-25:])
    assert "Backend B200_0" in out or "B200_0" in out, tail
    m = re.search(r"(\d+)/(\d+) tests passed", out)
    assert m, tail
    ok, total = int(m.group(1)), int(m.group(2))
    fails = [l for l in out.splitlines() if "FAIL" in l or "NMSE" in l][:10]
    assert rc == 0 and ok == total, (ok, total, fails)
    n_ok = len(re.findall(r": OK", out))
    assert n_ok > 0 or op in ("SILU",), f"backend supported no {op} case: nothing was exercised\n{tail}"


def test_backend_perf_mode_mul_mat(cuda):
    """test-backend-ops perf (m=4096, k=14336, n=1: tests/test-backend-ops.cpp:3703-3709) runs on the "B200" ggml backend and prints GB/s."""
    rc, out = run_tbo(["perf", "-b", "B200_0", "-o", "MUL_MAT"], timeout=600)
    assert rc == 0, out[-2000:]
    lines = [l for l in out.splitlines() if "q4_K" in l and "n=1," in l]
    assert lines, out[-2000:]
    print("\n".join(lines))
