"""TEST INFRASTRUCTURE — builds oracle/_ref/kaolin_ref_point_mesh_C.so, the reference's point-to-mesh
distance operators (``_C.metrics.unbatched_triangle_distance_{forward,backward}_cuda``, the CUDA path of
``point_to_mesh_distance``).

Compiles, in place and unmodified,

    kaolin/csrc/metrics/unbatched_triangle_distance.cpp, unbatched_triangle_distance_cuda.cu

plus oracle/ref_point_mesh_shim.cpp, with the flags of the check_sign recipe (-O3, -DWITH_CUDA, sm_90a).
The object of unbatched_triangle_distance_cuda.cu is kept next to the .so for SASS inspection: the
arithmetic of kaolin_b200/csrc/point_mesh_distance.cu follows the FMA contraction read from it.
Only usable where the reference's sources exist; elsewhere the prebuilt .so under oracle/_ref is used.
"""
import os
import subprocess
import sys
import sysconfig

from .build_ref import OUT, REF

HERE = os.path.dirname(os.path.abspath(__file__))
NAME = "kaolin_ref_point_mesh_C"


def build(force=False, verbose=True):
    so = os.path.join(OUT, NAME + ".so")
    csrc = os.path.join(REF, "kaolin", "csrc")
    if not os.path.isdir(csrc):
        return so if os.path.exists(so) else None
    srcs = [os.path.join(csrc, "metrics/unbatched_triangle_distance.cpp"),
            os.path.join(csrc, "metrics/unbatched_triangle_distance_cuda.cu"),
            os.path.join(HERE, "ref_point_mesh_shim.cpp")]
    if not force and os.path.exists(so) and all(os.path.getmtime(so) >= os.path.getmtime(s) for s in srcs):
        return so
    import torch
    from torch.utils import cpp_extension as ce
    os.makedirs(OUT, exist_ok=True)
    inc = [f"-I{p}" for p in ce.include_paths("cuda")] + [f"-I{sysconfig.get_paths()['include']}", f"-I{csrc}"]
    common = ["-O3", "-DWITH_CUDA", "-DTHRUST_IGNORE_CUB_VERSION_CHECK", f"-DTORCH_EXTENSION_NAME={NAME}",
              "-DTORCH_API_INCLUDE_EXTENSION_H", f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}",
              "-std=c++17"] + inc
    objs, procs = [], []
    for s in srcs:
        o = os.path.join(OUT, "point_mesh_" + os.path.basename(s) + ".o")
        objs.append(o)
        if s.endswith(".cu"):
            cmd = ["nvcc", "-c", s, "-o", o, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
                   "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xptxas", "-v"] + common
        else:
            cmd = ["g++", "-c", s, "-o", o, "-fPIC"] + common
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        log = p.communicate()[0]
        if p.returncode != 0:
            raise RuntimeError("reference compile failed: " + " ".join(cmd) + "\n" + log)
        if verbose and "ptxas" in log:
            print("\n".join(l for l in log.splitlines() if "Used" in l or "spill" in l))
    libdirs = ce.library_paths("cuda")
    subprocess.check_call(["g++", "-shared", "-o", so] + objs + [f"-L{d}" for d in libdirs]
                          + [f"-Wl,-rpath,{d}" for d in libdirs]
                          + ["-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
                             "-lcudart"])
    for o in objs:
        if o.endswith(".cpp.o"):
            os.remove(o)   # keep unbatched_triangle_distance_cuda.cu.o for SASS inspection
    return so


def load():
    """Import the prebuilt reference extension, or None when it has not been built."""
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)
    so = os.path.join(OUT, NAME + ".so")
    if not os.path.exists(so):
        return None
    spec = importlib.util.spec_from_file_location(NAME, so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    build(force="--force" in sys.argv)
