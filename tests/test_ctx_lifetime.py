"""Resource lifetime of the library: the whole library compiled over the CUDA-on-CPU shim (tests/cuda_emu) and a C driver
(tests/cuda_emu/lifetime_driver.c), both with AddressSanitizer.  The driver creates and destroys contexts, makes each allocation of
rgbl_create and of the lazily allocating entry points fail in turn, and expects RGBL_E_CUDA, then a retry on the same context with
a fresh context's outputs.  LeakSanitizer reports anything left allocated at exit.  PoseOptimization and the tracking chain are not
emulated: their streams, events, pinned staging and graphs are covered by the GPU suite only."""
import os
import subprocess
from pathlib import Path

import pytest

from cuda_emu import build

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent


def _run(cmd, **kw):
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1")
    return subprocess.run(cmd, capture_output=True, text=True, env=env, **kw)


def test_ctx_lifetime_under_address_sanitizer(tmp_path):
    leak = tmp_path / "leak.c"
    leak.write_text("#include <stdlib.h>\nvoid* volatile p;\nint main(void) { p = malloc(64); p = 0; return 0; }\n")
    subprocess.run(["gcc", "-fsanitize=address", "-o", str(tmp_path / "leak"), str(leak)], check=True)
    probe = _run([str(tmp_path / "leak")])
    if "LeakSanitizer: detected memory leaks" not in probe.stderr:
        pytest.skip("LeakSanitizer cannot run here: a program that leaks on purpose is not reported (" + probe.stderr.strip()[-200:] + ")")

    lib = build.build_full(sanitize="address")
    driver = tmp_path / "lifetime_driver"
    subprocess.run(["gcc", "-std=c99", "-O1", "-g", "-fsanitize=address", f"-I{ROOT / 'include'}", str(HERE / "cuda_emu" / "lifetime_driver.c"),
                    f"-L{lib.parent}", "-lrgbl_b200_emu", f"-Wl,-rpath,{lib.parent}", "-lz", "-lm", "-o", str(driver)], check=True)
    r = _run([str(driver)], timeout=1200)
    report = r.stdout + r.stderr
    assert r.returncode == 0, report[-6000:]
    assert "Sanitizer" not in r.stderr, report[-6000:]
    assert "0 failed checks" in r.stdout
