"""Builds libmeb200.so (the C-ABI library) in-tree with nvcc for sm_90a (H100).

    python minkowskiengine_b200/csrc/build.py [--force] [--verbose]

One `nvcc -c` per translation unit (parallel), then one `nvcc -shared` link.  The host
compiler is pinned to /usr/bin/g++ (the image's default CXX links libstdc++ statically,
see DESIGN.md "Toolchain").  The .so is git-ignored but travels to the GPU box.
"""
import concurrent.futures as cf
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
# A/B builds for kernel experiments: MEB200_BUILD_SUFFIX=_x MEB200_BUILD_DEFINES=-DNAME=VALUE
# writes libmeb200_x.so next to the default library (selected at run time with MEB200_LIB).
SUFFIX = os.environ.get("MEB200_BUILD_SUFFIX", "")
DEFINES = os.environ.get("MEB200_BUILD_DEFINES", "").split()
SO = os.path.join(HERE, f"libmeb200{SUFFIX}.so")
OBJ = os.path.join(HERE, f"build{SUFFIX}")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-lineinfo", "-std=c++17", "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr"]


def _deps_mtime():
    hdrs = glob.glob(os.path.join(HERE, "*.cuh")) + glob.glob(os.path.join(HERE, "*.h"))
    hdrs.append(os.path.join(HERE, "..", "..", "include", "meb200.h"))
    return max(os.path.getmtime(h) for h in hdrs)


def build(force=False, verbose=False):
    srcs = sorted(glob.glob(os.path.join(HERE, "*.cu")))
    os.makedirs(OBJ, exist_ok=True)
    hdr_t = _deps_mtime()
    jobs = []
    for s in srcs:
        o = os.path.join(OBJ, os.path.basename(s)[:-3] + ".o")
        stale = force or not os.path.isfile(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_t)
        jobs.append((s, o, stale))

    def cc(job):
        s, o, stale = job
        if stale:
            cmd = [NVCC, *ARCH, *FLAGS, *DEFINES, "-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd), flush=True)
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {s}:\n{r.stdout}\n{r.stderr}")
        return o

    with cf.ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(cc, jobs))
    need_link = force or not os.path.isfile(SO) or any(j[2] for j in jobs) or \
        any(os.path.getmtime(o) > os.path.getmtime(SO) for o in objs)
    if need_link:
        cmd = [NVCC, *ARCH, "-shared", "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fPIC", *objs,
               "-o", SO, "-lcudart"]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
