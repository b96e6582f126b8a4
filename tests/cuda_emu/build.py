"""TEST INFRASTRUCTURE: builds tests/cuda_emu/build/librgbl_b200_emu.so = the whole library (every .cu / .cpp of csrc/Makefile) compiled
by g++ against the CUDA-on-CPU shim in this directory (device code paths, one OS thread per CUDA thread), together with every .cpp of this
directory: the shim's runtime, its stubs, and the emu_* entry points that run single kernels through their launchers.  It exports the C ABI
of include/rgbl_b200.h, so the -m gpu parity tests can run on the CPU (RGBL_LIB_PATH, see orb_slam3_rgbl_b200/_lib.py), and the emu_*
functions of the tests/test_cuda_emu*.py files.  Source transformations (text only, into a scratch directory): kernel launches
`k<<<cfg>>>(args);` -> emu::run(emu::cfg(cfg), [&]{ k(args); }); and dynamic shared-memory declarations -> a static buffer."""
from __future__ import annotations

import re
import shutil
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
CSRC = ROOT / "orb_slam3_rgbl_b200" / "csrc"
BUILD = HERE / "build"


def _cluster_transform(text: str) -> str:
    """A file with a __cluster_dims__ kernel: its CTAs run concurrently, so every __shared__ variable becomes a slot of the emulated
    cluster shared window (cuda_runtime.h, emu::cluster_shared), its launch runs as clusters, and the DSMEM / mbarrier PTX becomes
    the shim's model of it (tx-count and phase parity kept)."""
    ids = iter(range(1 << 20))

    def decl(m):
        out = []
        for d in m.group(2).split(","):
            name, dims = re.fullmatch(r"\s*(\w+)((?:\[[^\]]+\])*)\s*", d).groups()
            out.append(f"auto& {name} = emu::cluster_shared<{m.group(1)}{dims}, {next(ids)}>();")
        return " ".join(out)
    text = re.sub(r"__shared__ (?:__align__\(\d+\) )?((?:unsigned )?(?:long long|\w+)) ([^;]+);", decl, text)
    for size, name in re.findall(r"__cluster_dims__\((\w+), 1, 1\)[^(]*\([^)]*\) (\w+)\(", text):
        text = re.sub(rf"\blaunch_kernel\({name},", f"emu::next_launch_cluster({size}), launch_kernel({name},", text)
    text = re.sub(r'asm volatile\("mapa\.shared::cluster\.u32 %0, %1, %2;" : "=r"\((\w+)\) : "r"\((\w+)\), "r"\((\w+)\)\);',
                  r"\1 = emu::mapa(\2, \3);", text)
    text = re.sub(r'asm volatile\("mbarrier\.init\.shared::cta\.b64 \[%0\], (\d+);" :: "r"\((.*)\)\);', r"emu::mbar_init(\2, \1);", text)
    text = text.replace('asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");', "std::atomic_thread_fence(std::memory_order_seq_cst);")
    text = re.sub(r'asm volatile\("mbarrier\.arrive\.expect_tx\.shared::cta\.b64 _, \[%0\], %1;" :: "r"\((.*?)\), "r"\((.*)\) : "memory"\);',
                  r"emu::mbar_arrive_expect_tx(\1, \2);", text)
    text = re.sub(r'asm volatile\("st\.async\.weak\.shared::cluster\.mbarrier::complete_tx::bytes\.b64 \[%0\], %1, \[%2\];"\s*'
                  r':: "r"\((.*?)\), "l"\((.*?)\), "r"\((.*?)\) : "memory"\);', r"emu::st_async_b64(\1, \2, \3);", text)
    text = re.sub(r'asm volatile\("\{ \.reg \.pred p; mbarrier\.try_wait\.parity\.shared::cta\.b64 p, \[%1\], %2; selp\.u32 %0, 1, 0, p; \}"\s*'
                  r': "=r"\((\w+)\) : "r"\((\w+)\), "r"\((\w+)\) : "memory"\);', r"\1 = emu::mbar_try_wait_parity(\2, \3);", text)
    return text


def _transform(text: str) -> str:
    cluster = "__cluster_dims__" in text
    if cluster:
        text = _cluster_transform(text)
    text = re.sub(r"extern __shared__ (?:__align__\(16\) )?(\w+(?: \w+)*) (\w+)\[\];", r"alignas(16) static \1 \2[emu::kDynSmem / sizeof(\1)];", text)
    text = re.sub(r"(\w+(?:<[^<>;]*>)?)<<<(.+?)>>>\((.*?)\);", r"emu::run(emu::cfg(\2), [&]() { \1(\3); });", text, flags=re.S)
    # the two approximate FP64 MUFU seeds of the LM kernel (results have 32 zero low mantissa bits, PTX ISA "rcp.approx.ftz.f64")
    text = re.sub(r'asm\("rcp\.approx\.ftz\.f64 %0, %1;" : "=d"\((\w+)\) : "d"\((\w+)\)\);', r"\1 = emu::approx64(1.0 / \2);", text)
    text = re.sub(r'asm\("rsqrt\.approx\.ftz\.f64 %0, %1;" : "=d"\((\w+)\) : "d"\((\w+)\)\);', r"\1 = emu::approx64(1.0 / std::sqrt(\2));", text)
    text = text.replace('#include "../../include/rgbl_b200.h"', f'#include "{ROOT}/include/rgbl_b200.h"')
    left = [l.strip() for l in text.splitlines() if re.search(r"\basm\b", l.split("//")[0])]
    if cluster and left:             # a cluster kernel whose PTX is not modelled must not compile into something else
        raise RuntimeError("inline PTX the shim does not model:\n" + "\n".join(left))
    return text


FULL_SRCS = ["api.cu", "api_track.cu", "quadtree_kernels.cu", "orb_kernels.cu", "fast_strip_kernels.cu", "describe_warp_kernels.cu", "depth_kernels.cu",
             "depth_dilate_v2.cu", "stereo_kernels.cu", "match_kernels.cu", "bow_kernels.cu", "api_bow.cu", "api_ba.cu", "api_mapping.cu", "chain_kernels.cu", "png_kernels.cu",
             "pose_kernels.cu", "quadtree_host.cpp", "host_tables.cpp"]
# pose_kernels.cu (PoseOptimization) is a thread-block cluster exchanging partial sums with st.async + mbarrier: _cluster_transform
# runs all CTAs of its cluster at once and models the exchange; build_full(defines=["-DPOSE_CTAS=8", "-DPOSE_THREADS=128"]) builds
# it at another cluster shape.  level_tma_kernels.cu (TMA tensor maps) is not emulated: emu_stubs.cpp.


def build_full(defines=(), sanitize: str | None = None) -> Path:
    """The library over the shim, rebuilt when any of its sources is newer than it.  defines: extra compiler flags; sanitize ("address" |
    "thread"): builds with -fsanitize=....  Without either the library is build/librgbl_b200_emu.so; any other flag set builds into a
    subdirectory of build/ named after its flags, so a cached library always matches the flags it was asked for."""
    from concurrent.futures import ThreadPoolExecutor
    san = ["-fsanitize=" + sanitize] if sanitize else []
    extra = list(defines) + san
    out_dir = BUILD / "_".join(f.lstrip("-") for f in extra) if extra else BUILD
    lib = out_dir / "librgbl_b200_emu.so"
    hdrs = [f.name for f in CSRC.iterdir() if f.suffix in (".h", ".cuh", ".inc")]
    entries = sorted(HERE.glob("*.cpp"))
    srcs = [CSRC / f for f in FULL_SRCS + hdrs] + entries + [HERE / "cuda_runtime.h", HERE / "cooperative_groups.h", Path(__file__)]
    if lib.exists() and all(lib.stat().st_mtime > s.stat().st_mtime for s in srcs):
        return lib
    full = out_dir / "full"
    if full.exists():
        shutil.rmtree(full)
    full.mkdir(parents=True)
    for f in FULL_SRCS + hdrs:
        out = full / ((f[:-3] + ".emu.cpp") if f.endswith(".cu") else f)
        out.write_text(_transform((CSRC / f).read_text()))
    # -fno-gnu-unique: two of these libraries (other cluster shapes) loaded in one process must not share the static locals of inline
    # functions (emu::cluster_shared offsets), which g++ would otherwise unify across libraries even under RTLD_LOCAL
    flags = ["-std=c++20", "-O1", "-g", "-pthread", "-fPIC", "-fno-gnu-unique", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", f"-I{HERE}", f"-I{full}",
             "-include", str(HERE / "cuda_runtime.h"), "-DRGBL_TESTING_EXPORTS"] + extra       # the shim first: __CUDA_ARCH__ must be set before any header
    units = [full / ((f[:-3] + ".emu.cpp") if f.endswith(".cu") else f) for f in FULL_SRCS] + entries

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


if __name__ == "__main__":
    import sys
    print(build_full(sanitize=sys.argv[1] if len(sys.argv) > 1 else None))
