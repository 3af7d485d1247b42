#!/usr/bin/env python3
"""In-tree native build for blackbird_b200.

Generates build/build.ninja and runs ninja.  Produces
  blackbird_b200/_bb<EXT_SUFFIX>   single pybind11 module: C++20 control plane + sm_90a data plane
  bin/bb-keystone bin/bb-worker bin/bb-coord bin/bb-cli bin/bb-bench bin/bb-tests

All CUDA is compiled for sm_90a only (`-gencode arch=compute_90a,code=sm_90a -lineinfo`);
nvcc cross-compiles without a GPU.  cudart is linked statically and the driver API is
resolved at runtime, so the module imports on a CPU-only box.
"""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
import sys
import sysconfig

ROOT = os.path.dirname(os.path.abspath(__file__))
# Sanitizer builds (BB_SANITIZE=asan|tsan) are kept apart from the production build: objects in build/<san>/, the
# extension and the binaries in build/<san>/out/{blackbird_b200,bin} (the package directory there is a tree of links
# to the python sources).  Run the suite against them with
#   BB_PKG_ROOT=build/asan/out BB_BIN_DIR=$PWD/build/asan/out/bin python -m pytest tests -m "not gpu"
SAN = os.environ.get("BB_SANITIZE", "")
BUILD = os.path.join(ROOT, "build", SAN) if SAN else os.path.join(ROOT, "build")
OUT = os.path.join(BUILD, "out") if SAN else ROOT
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")

CXXFLAGS = "-std=c++20 -O2 -g1 -fPIC -Wall -Wextra -Wno-unused-parameter -Wno-missing-field-initializers -pthread"
NVCCFLAGS = (
    "-std=c++20 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a "
    "-Xcompiler -fPIC -Xcompiler -Wall -Xptxas -v --expt-relaxed-constexpr -Wno-deprecated-gpu-targets"
)


def _san_flags() -> str:
    san = SAN
    if san == "asan":
        return " -fsanitize=address,undefined -fno-omit-frame-pointer"
    if san == "tsan":
        return " -fsanitize=thread -fno-omit-frame-pointer"
    return ""


def _rel(p: str) -> str:
    return os.path.relpath(p, BUILD)


def generate() -> str:
    import pybind11

    os.makedirs(BUILD, exist_ok=True)
    ext = sysconfig.get_config_var("EXT_SUFFIX")
    pyinc = sysconfig.get_paths()["include"]
    incs = f"-I{ROOT}/csrc -I{ROOT} -I{CUDA_HOME}/include"
    pyincs = f"-I{pybind11.get_include()} -I{pyinc}"
    san = _san_flags()

    core_src = sorted(
        f
        for d in ("common", "alloc", "coord", "net", "rpc", "keystone", "worker", "client")
        for f in glob.glob(os.path.join(ROOT, "csrc", d, "*.cpp"))
    )
    fabric_src = sorted(glob.glob(os.path.join(ROOT, "csrc", "fabric", "*.cpp")))
    cu_src = sorted(glob.glob(os.path.join(ROOT, "csrc", "kernels", "*.cu")))
    py_src = sorted(glob.glob(os.path.join(ROOT, "csrc", "py", "*.cpp")))
    app_src = sorted(glob.glob(os.path.join(ROOT, "apps", "*.cpp")))
    example_src = sorted(glob.glob(os.path.join(ROOT, "examples", "*.cpp")))  # -> bin/bb-example-<name>
    tool_cu_src = sorted(glob.glob(os.path.join(ROOT, "bench", "*.cu")))  # stand-alone CUDA tools -> bin/bb-<name>

    lines = [
        "ninja_required_version = 1.5",
        f"cxxflags = {CXXFLAGS}{san} {incs}",
        f"nvccflags = {NVCCFLAGS} {incs}",
        f"pyincs = {pyincs}",
        "rule cxx",
        "  command = g++ -MMD -MF $out.d $cxxflags $extra -c $in -o $out",
        "  depfile = $out.d",
        "  deps = gcc",
        "  description = CXX $in",
        "rule nvcc",
        f"  command = {NVCC} $nvccflags -MD -MF $out.d -c $in -o $out 2> $out.ptxas.log || (cat $out.ptxas.log; false)",
        "  depfile = $out.d",
        "  deps = gcc",
        "  description = NVCC $in",
        "rule link_so",
        f"  command = g++ -shared -o $out $in -L{CUDA_HOME}/lib64 -lcudart_static -ldl -lrt -pthread{san}",
        "  description = LINK $out",
        "rule link_cuda_exe",
        f"  command = g++ -o $out $in -L{CUDA_HOME}/lib64 -lcudart_static -L{CUDA_HOME}/lib64/stubs -lcuda -ldl -lrt -pthread",
        "  description = LINK $out",
        "rule link_exe",
        f"  command = g++ -o $out $in -L{CUDA_HOME}/lib64 -lcudart_static -ldl -lrt -pthread{san}",
        "  description = LINK $out",
        "",
    ]

    def obj(src: str) -> str:
        return os.path.join("obj", os.path.relpath(src, ROOT).replace("/", "_") + ".o")

    lib_objs = []
    for s in core_src + fabric_src:
        o = obj(s)
        lib_objs.append(o)
        lines.append(f"build {o}: cxx {_rel(s)}")
    for s in cu_src:
        o = obj(s)
        lib_objs.append(o)
        lines.append(f"build {o}: nvcc {_rel(s)}")
    py_objs = []
    for s in py_src:
        o = obj(s)
        py_objs.append(o)
        lines.append(f"build {o}: cxx {_rel(s)}")
        lines.append("  extra = $pyincs -fvisibility=hidden")
    mod = _rel(os.path.join(OUT, "blackbird_b200", "_bb" + ext))
    lines.append(f"build {mod}: link_so {' '.join(py_objs + lib_objs)}")
    targets = [mod]
    for s in app_src:
        o = obj(s)
        lines.append(f"build {o}: cxx {_rel(s)}")
        name = os.path.splitext(os.path.basename(s))[0].replace("_", "-")
        exe = _rel(os.path.join(OUT, "bin", name))
        lines.append(f"build {exe}: link_exe {o} {' '.join(lib_objs)}")
        targets.append(exe)
    for s in example_src:
        o = obj(s)
        lines.append(f"build {o}: cxx {_rel(s)}")
        name = "bb-example-" + os.path.splitext(os.path.basename(s))[0].replace("_", "-")
        exe = _rel(os.path.join(OUT, "bin", name))
        lines.append(f"build {exe}: link_exe {o} {' '.join(lib_objs)}")
        targets.append(exe)
    for s in tool_cu_src:
        o = obj(s)
        lines.append(f"build {o}: nvcc {_rel(s)}")
        name = "bb-" + os.path.splitext(os.path.basename(s))[0].replace("_", "-")
        exe = _rel(os.path.join(OUT, "bin", name))
        lines.append(f"build {exe}: link_cuda_exe {o}")
        targets.append(exe)
    lines.append(f"default {' '.join(targets)}")
    path = os.path.join(BUILD, "build.ninja")
    content = "\n".join(lines) + "\n"
    old = open(path).read() if os.path.exists(path) else None
    if old != content:
        with open(path, "w") as f:
            f.write(content)
    return path


def build(verbose: bool = False, targets: list[str] | None = None) -> None:
    generate()
    os.makedirs(os.path.join(OUT, "bin"), exist_ok=True)
    if OUT != ROOT:  # link the python sources next to the sanitized extension
        pkg_src, pkg_dst = os.path.join(ROOT, "blackbird_b200"), os.path.join(OUT, "blackbird_b200")
        os.makedirs(pkg_dst, exist_ok=True)
        for name in os.listdir(pkg_src):
            if name.startswith("_bb.") or name == "__pycache__":
                continue
            dst = os.path.join(pkg_dst, name)
            if not os.path.lexists(dst):
                os.symlink(os.path.join(pkg_src, name), dst)
    ninja = shutil.which("ninja")
    if ninja is None:
        raise RuntimeError("ninja not found")
    cmd = [ninja, "-C", BUILD]
    if verbose:
        cmd.append("-v")
    if targets:
        cmd += targets
    r = subprocess.run(cmd)
    if r.returncode != 0:
        raise RuntimeError("native build failed")


if __name__ == "__main__":
    build(verbose="-v" in sys.argv)
