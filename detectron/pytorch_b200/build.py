"""In-tree build of libb200_roi_ops.so (sm_90a only, nvcc; no torch headers -- pure C ABI).

    python -m detectron.pytorch_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU, so this also runs on a machine without one; the resulting
.so is git-ignored.
"""
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.environ.get("B200_ROI_OPS_LIB") or os.path.join(PKG_DIR, "libb200_roi_ops.so")     # override: A/B builds
INCLUDE = os.path.join(os.path.dirname(os.path.dirname(PKG_DIR)), "include")
CSRC_COMPAT = os.path.join(PKG_DIR, "csrc_compat")
# the reference's launcher names on top of the C ABI (include/b200_ref_launchers.h): name -> extra nvcc defines
COMPAT_LIBS = {
    "libb200_ref_launchers.so": [],
    "libb200_ref_launchers_legacy.so": ["-DB200_REF_LEGACY_ROI_ALIGN"],
}

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--shared",
    # the kernels write every fusion explicitly with _rn intrinsics; keep the default -fmad=true,
    # -prec-div=true, -prec-sqrt=true, no --use_fast_math (numerics must match the reference).
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps():
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    deps.append(os.path.join(INCLUDE, "b200_roi_ops.h"))
    deps.append(os.path.join(INCLUDE, "b200_ref_launchers.h"))
    deps.append(os.path.join(CSRC_COMPAT, "ref_launchers.cu"))
    return deps


def compat_lib_path(name):
    return os.path.join(os.path.dirname(LIB_PATH), name)


def needs_build():
    outs = [LIB_PATH] + ([] if os.environ.get("B200_ROI_OPS_LIB") else [compat_lib_path(n) for n in COMPAT_LIBS])
    if not all(os.path.exists(o) for o in outs):
        return True
    t = min(os.path.getmtime(o) for o in outs)
    return any(os.path.getmtime(d) > t for d in _deps())


def find_nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library.  Returns the library path."""
    if not force and not needs_build():
        return LIB_PATH
    nvcc = find_nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libb200_roi_ops.so (set $NVCC)")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-I", INCLUDE, "-o", LIB_PATH + ".tmp"] + sources()
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libb200_roi_ops.so (exit %d)" % res.returncode)
    os.replace(LIB_PATH + ".tmp", LIB_PATH)
    # compatibility libraries: tiny, link against the main library next to them (rpath $ORIGIN)
    libdir, libname = os.path.split(LIB_PATH)
    for name, defines in COMPAT_LIBS.items():
        if os.environ.get("B200_ROI_OPS_LIB"):
            break                                          # A/B build of the main library only
        out = compat_lib_path(name)
        cmd = [nvcc] + NVCC_FLAGS + defines + ["-I", INCLUDE, "-o", out + ".tmp", os.path.join(CSRC_COMPAT, "ref_launchers.cu"),
                                                 "-L", libdir, "-l:" + libname, "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if verbose or res.returncode != 0:
            sys.stderr.write(res.stdout)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed building %s (exit %d)" % (name, res.returncode))
        os.replace(out + ".tmp", out)
    return LIB_PATH


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
