"""TEST INFRASTRUCTURE: builds tests/cuda_emu/build/libcuda_emu.so = a few of the library's .cu files compiled by g++ against the
CUDA-on-CPU shim in this directory (device code paths, one OS thread per CUDA thread).  Source transformations (text only,
into a scratch directory): kernel launches `k<<<cfg>>>(args);` -> emu::run(emu::cfg(cfg), [&]{ k(args); }); and dynamic
shared-memory declarations -> a static buffer."""
from __future__ import annotations

import re
import shutil
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
CSRC = ROOT / "orb_slam3_rgbl_b200" / "csrc"
BUILD = HERE / "build"
LIB = BUILD / "libcuda_emu.so"
KERNEL_FILES = ["orb_kernels.cu", "fast_strip_kernels.cu", "describe_warp_kernels.cu", "quadtree_kernels.cu", "depth_kernels.cu", "depth_dilate_v2.cu"]
HEADERS = ["fast_strip.cuh", "describe_warp.cuh", "quadtree_block.cuh", "rgbl_device.cuh", "rgbl_kernels.h", "rgbl_internal.h", "rgbl_testing.h",
           "orb_pattern_31.inc"]
HOST_FILES = ["host_tables.cpp", "quadtree_host.cpp"]


def _transform(text: str) -> str:
    text = re.sub(r"extern __shared__ (?:__align__\(16\) )?(\w+(?: \w+)*) (\w+)\[\];", r"alignas(16) static \1 \2[emu::kDynSmem / sizeof(\1)];", text)
    text = re.sub(r"(\w+(?:<[^<>;]*>)?)<<<(.+?)>>>\((.*?)\);", r"emu::run(emu::cfg(\2), [&]() { \1(\3); });", text, flags=re.S)
    # the two approximate FP64 MUFU seeds of the LM kernel (results have 32 zero low mantissa bits, PTX ISA "rcp.approx.ftz.f64")
    text = re.sub(r'asm\("rcp\.approx\.ftz\.f64 %0, %1;" : "=d"\((\w+)\) : "d"\((\w+)\)\);', r"\1 = emu::approx64(1.0 / \2);", text)
    text = re.sub(r'asm\("rsqrt\.approx\.ftz\.f64 %0, %1;" : "=d"\((\w+)\) : "d"\((\w+)\)\);', r"\1 = emu::approx64(1.0 / std::sqrt(\2));", text)
    text = text.replace('#include "../../include/rgbl_b200.h"', f'#include "{ROOT}/include/rgbl_b200.h"')
    return text


def build(force: bool = False) -> Path:
    srcs = [CSRC / f for f in KERNEL_FILES + HEADERS + HOST_FILES] + [HERE / "cuda_runtime.h", HERE / "emu_runtime.cpp", HERE / "emu_entry.cpp", Path(__file__)]
    if LIB.exists() and not force and all(LIB.stat().st_mtime > s.stat().st_mtime for s in srcs):
        return LIB
    if BUILD.exists():
        shutil.rmtree(BUILD)
    BUILD.mkdir(parents=True)
    for f in KERNEL_FILES + HEADERS + HOST_FILES:
        out = BUILD / (f[:-3] + ".emu.cpp" if f.endswith(".cu") else f)
        out.write_text(_transform((CSRC / f).read_text()))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-DRGBL_TESTING_EXPORTS",
           f"-I{HERE}", f"-I{BUILD}", "-o", str(LIB), str(HERE / "emu_entry.cpp"), str(HERE / "emu_runtime.cpp"), *[str(BUILD / f) for f in HOST_FILES]]
    subprocess.run(cmd, check=True)
    return LIB


FULL_LIB = BUILD / "librgbl_b200_emu.so"
FULL_SRCS = ["api.cu", "api_track.cu", "quadtree_kernels.cu", "orb_kernels.cu", "fast_strip_kernels.cu", "describe_warp_kernels.cu", "depth_kernels.cu",
             "depth_dilate_v2.cu", "stereo_kernels.cu", "match_kernels.cu", "bow_kernels.cu", "api_bow.cu", "api_ba.cu", "api_mapping.cu", "chain_kernels.cu", "png_kernels.cu",
             "quadtree_host.cpp", "host_tables.cpp"]
# pose_kernels.cu is NOT emulated since round 2: the LM kernel is a 4-CTA thread-block cluster exchanging partial sums with
# st.async + mbarrier (PTX); emu_stubs.cpp aborts with a message if the emulated library reaches PoseOptimization.


def build_full(force: bool = False, defines=(), sanitize: str | None = None, out_dir: Path | None = None) -> Path:
    """The WHOLE library (every .cu / .cpp of csrc/Makefile) against the shim: build/librgbl_b200_emu.so exports the C ABI of
    include/rgbl_b200.h, so the -m gpu parity tests can run on the CPU (RGBL_LIB_PATH, see orb_slam3_rgbl_b200/_lib.py).
    sanitize ("address" | "thread") builds with -fsanitize=...; out_dir: where the library and its objects go (default build/)."""
    from concurrent.futures import ThreadPoolExecutor
    out_dir = Path(out_dir) if out_dir else BUILD
    lib = out_dir / FULL_LIB.name
    hdrs = [f.name for f in CSRC.iterdir() if f.suffix in (".h", ".cuh", ".inc")]
    srcs = [CSRC / f for f in FULL_SRCS + hdrs] + [HERE / "cuda_runtime.h", HERE / "emu_runtime.cpp", Path(__file__)]
    if lib.exists() and not force and all(lib.stat().st_mtime > s.stat().st_mtime for s in srcs):
        return lib
    full = out_dir / "full"
    if full.exists():
        shutil.rmtree(full)
    full.mkdir(parents=True)
    for f in FULL_SRCS + hdrs:
        out = full / ((f[:-3] + ".emu.cpp") if f.endswith(".cu") else f)
        out.write_text(_transform((CSRC / f).read_text()))
    san = ["-fsanitize=" + sanitize] if sanitize else []
    flags = ["-std=c++20", "-O1", "-g", "-pthread", "-fPIC", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", f"-I{HERE}", f"-I{full}",
             "-include", str(HERE / "cuda_runtime.h"), "-DRGBL_TESTING_EXPORTS"] + list(defines) + san       # the shim first: __CUDA_ARCH__ must be set before any header
    units = [full / ((f[:-3] + ".emu.cpp") if f.endswith(".cu") else f) for f in FULL_SRCS] + [HERE / "emu_runtime.cpp", HERE / "emu_stubs.cpp"]

    def cc(u):
        o = full / (u.name + ".o")
        r = subprocess.run(["g++", *flags, "-c", "-o", str(o), str(u)], capture_output=True, text=True)
        if r.returncode:
            return RuntimeError(f"{u.name}:\n" + "\n".join(l for l in r.stderr.splitlines() if "error" in l)[:2500])
        return o
    with ThreadPoolExecutor(8) as ex:
        objs = list(ex.map(cc, units))
    errs = [o for o in objs if isinstance(o, Exception)]
    if errs:
        raise RuntimeError("\n".join(str(e) for e in errs))
    subprocess.run(["g++", "-shared", "-pthread", *san, "-o", str(lib), *map(str, objs), "-lz"], check=True)
    return lib


TLM_CHECK = BUILD / "tlm_check"


def build_tlm_check(force: bool = False) -> Path:
    """tlm_check.cpp + chain_kernels.cu against the shim -> an executable comparing the multi-CTA TrackLocalMap glue kernels with a
    serial restatement (tests/test_cuda_emu.py::test_tlm_kernels_device_path)."""
    hdrs = [f.name for f in CSRC.iterdir() if f.suffix in (".h", ".cuh", ".inc")]
    srcs = [CSRC / f for f in ["chain_kernels.cu"] + hdrs] + [HERE / "cuda_runtime.h", HERE / "emu_runtime.cpp", HERE / "tlm_check.cpp", Path(__file__)]
    if TLM_CHECK.exists() and not force and all(TLM_CHECK.stat().st_mtime > s.stat().st_mtime for s in srcs):
        return TLM_CHECK
    d = BUILD / "tlm"
    if d.exists():
        shutil.rmtree(d)
    d.mkdir(parents=True)
    for f in ["chain_kernels.cu"] + hdrs:
        out = d / ((f[:-3] + ".emu.cpp") if f.endswith(".cu") else f)
        out.write_text(_transform((CSRC / f).read_text()))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", f"-I{HERE}", f"-I{d}", "-include", str(HERE / "cuda_runtime.h"),
           "-o", str(TLM_CHECK), str(HERE / "tlm_check.cpp"), str(d / "chain_kernels.emu.cpp"), str(HERE / "emu_runtime.cpp")]
    subprocess.run(cmd, check=True)
    return TLM_CHECK


if __name__ == "__main__":
    import sys
    if len(sys.argv) > 1 and sys.argv[1] == "full":
        print(build_full(force=True))
        sys.exit(0)
    print(build(force=True))
