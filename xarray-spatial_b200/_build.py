"""Builds libxrs_b200.so in-tree with nvcc for the H100 (sm_90a); the package loads it from
next to its sources."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libxrs_b200.so")
SOURCES = ["lib_core.cu", "surface.cu", "multispectral.cu", "conv.cu", "box_stream.cu", "zonal_hash.cu", "hotspots.cu", "geodesic.cu", "proximity.cu", "viewshed.cu", "pathfinding.cu", "noise.cu", "classify.cu", "natural_breaks.cu", "zonal_regions.cu", "host.cu", "synth.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [
    "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false",  # no implicit FMA contraction: parity with the f64/f32 CPU arithmetic
    "-Xcompiler", "-fPIC", "-DXRS_BUILD",
]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    nvcc = os.environ.get("NVCC", "nvcc")
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "xrs_b200.h"))
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(o, [s] + headers):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd))
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError("nvcc failed on %s" % src)
    if force or procs or not os.path.exists(SO) or _newer(SO, objs):   # objects may have been rebuilt by hand
        cmd = [nvcc, "-shared"] + ARCH + ["-o", SO] + objs + ["-cudart", "static"]
        subprocess.check_call(cmd)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
