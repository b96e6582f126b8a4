"""Allocation failures of stereo rectification: the whole library over the CUDA-on-CPU shim and a C driver
(tests/cuda_emu/rectify_lifetime_driver.c), both with AddressSanitizer.  Each lazy allocation of the rectification (the fixed-point maps,
their float staging, the raw planes) fails once: the call returns RGBL_E_CUDA, the retry gives a
fresh context's outputs, and LeakSanitizer finds nothing left allocated."""
import importlib.util
import os
import subprocess
from pathlib import Path

import pytest

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent


def _run(cmd, **kw):
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1")
    return subprocess.run(cmd, capture_output=True, text=True, env=env, **kw)


def test_rectification_allocations_under_address_sanitizer(tmp_path):
    leak = tmp_path / "leak.c"
    leak.write_text("#include <stdlib.h>\nvoid* volatile p;\nint main(void) { p = malloc(64); p = 0; return 0; }\n")
    subprocess.run(["gcc", "-fsanitize=address", "-o", str(tmp_path / "leak"), str(leak)], check=True)
    if "LeakSanitizer: detected memory leaks" not in _run([str(tmp_path / "leak")]).stderr:
        pytest.skip("LeakSanitizer cannot run here: a program that leaks on purpose is not reported")
    spec = importlib.util.spec_from_file_location("cuda_emu_build", HERE / "cuda_emu" / "build.py")
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    lib = mod.build_full(force=True, sanitize="address", out_dir=tmp_path / "asan")
    driver = tmp_path / "rectify_lifetime_driver"
    subprocess.run(["gcc", "-std=c99", "-O1", "-g", "-fsanitize=address", f"-I{ROOT / 'include'}", str(HERE / "cuda_emu" / "rectify_lifetime_driver.c"),
                    f"-L{lib.parent}", "-lrgbl_b200_emu", f"-Wl,-rpath,{lib.parent}", "-lz", "-lm", "-o", str(driver)], check=True)
    r = _run([str(driver)], timeout=1200)
    report = r.stdout + r.stderr
    assert r.returncode == 0, report[-6000:]
    assert "Sanitizer" not in r.stderr, report[-6000:]
    assert "0 failed checks" in r.stdout
    # the maps (2), their staging and the raw planes, in both paths
    assert [int(line.rsplit(": ", 1)[1].split()[0]) for line in r.stdout.splitlines() if "allocations" in line] == [4, 4], r.stdout
