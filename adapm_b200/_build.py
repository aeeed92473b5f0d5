"""In-tree build of the native extension ``adapm_b200/_C*.so``.

Everything is compiled explicitly for sm_90a (``-gencode arch=compute_90a,code=sm_90a
-lineinfo``); nvcc cross-compiles without a GPU. The resulting ``.so`` sits next to the
Python sources, so the package imports straight from the repository tree.

    python -m adapm_b200._build            # incremental (ninja)
    python -m adapm_b200._build --force    # rebuild everything
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
BUILD = ROOT.parent / "build" / "adapm_b200"
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")

CXX_SOURCES = [
    "adapm/corpus.cc",
    "adapm/fabric.cc",
    "adapm/io.cc",
    "adapm/node.cc",
    "adapm/rpc.cc",
    "adapm/sampling.cc",
    "adapm/store_cpu.cc",
    "adapm/sync_engine.cc",
    "bindings.cc",
    "cuda/ops_bind.cc",
]
CUDA_SOURCES = [
    "cuda/device_mem.cu",
    "cuda/cuda_backend.cu",
    "cuda/fx_accum.cu",
]


def _cuda_sources():
    extra = sorted(p.relative_to(CSRC).as_posix() for p in (CSRC / "cuda").glob("ops_*.cu"))
    return CUDA_SOURCES + [e for e in extra if e not in CUDA_SOURCES]


def ext_path() -> Path:
    return ROOT / ("_C" + sysconfig.get_config_var("EXT_SUFFIX"))


def _ninja_file() -> str:
    import pybind11

    py_inc = sysconfig.get_paths()["include"]
    incs = f"-I{CSRC} -I{pybind11.get_include()} -I{py_inc} -I{CUDA_HOME}/include"
    cxxflags = f"-O3 -g1 -std=c++17 -fPIC -fvisibility=hidden -Wall -Wno-unused-function -pthread {incs}"
    nvflags = (
        "-O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=[sm_90a,compute_90a] "
        "--expt-relaxed-constexpr -Xcompiler -fPIC,-fvisibility=hidden,-pthread "
        f"-Xptxas -v {incs}"
    )
    lines = [
        "ninja_required_version = 1.3",
        f"cxxflags = {cxxflags}",
        f"nvflags = {nvflags}",
        "rule cxx",
        "  command = g++ -MMD -MF $out.d $cxxflags -c $in -o $out",
        "  depfile = $out.d",
        "  deps = gcc",
        "rule nvcc",
        f"  command = {CUDA_HOME}/bin/nvcc $nvflags -MD -MF $out.d -c $in -o $out > $out.log 2>&1 || (cat $out.log; false)",
        "  depfile = $out.d",
        "  deps = gcc",
        "rule link",
        f"  command = g++ -shared -o $out $in -L{CUDA_HOME}/lib64 -lcudart_static -ldl -lrt -lpthread",
    ]
    objs = []
    for s in CXX_SOURCES:
        o = BUILD / (s.replace("/", "_") + ".o")
        lines.append(f"build {o}: cxx {CSRC / s}")
        objs.append(str(o))
    for s in _cuda_sources():
        o = BUILD / (s.replace("/", "_") + ".o")
        lines.append(f"build {o}: nvcc {CSRC / s}")
        objs.append(str(o))
    lines.append(f"build {ext_path()}: link {' '.join(objs)}")
    # native (Python-free) application on the core API
    core = [o for o in objs if not (o.endswith("bindings.cc.o") or o.endswith("ops_bind.cc.o"))]
    app_o = BUILD / "apps_simple.cc.o"
    lines.append(f"build {app_o}: cxx {CSRC / 'apps/simple.cc'}")
    lines.append("rule linkexe")
    lines.append(f"  command = g++ -o $out $in -L{CUDA_HOME}/lib64 -lcudart_static -ldl -lrt -lpthread")
    lines.append(f"build {BUILD / 'adapm_simple'}: linkexe {app_o} {' '.join(core)}")
    lines.append(f"default {ext_path()} {BUILD / 'adapm_simple'}")
    return "\n".join(lines) + "\n"


def build(force: bool = False, verbose: bool = False) -> Path:
    BUILD.mkdir(parents=True, exist_ok=True)
    nf = BUILD / "build.ninja"
    text = _ninja_file()
    if force or not nf.exists() or nf.read_text() != text:
        nf.write_text(text)
    cmd = ["ninja", "-C", str(BUILD), "-f", str(nf)]
    if force:
        subprocess.run(cmd + ["-t", "clean"], check=False, stdout=subprocess.DEVNULL)
    if verbose:
        cmd.append("-v")
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("adapm_b200 native build failed")
    if verbose:
        print(r.stdout)
    return ext_path()


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
