"""In-tree build of the native libraries (no JIT cache: the .so files travel with the repo snapshot).

  dint_b200/lib/libdint_b200.so   CUDA kernels + C ABI (include/dint_b200.h), nvcc, sm_90a (H100) only
  dint_b200/lib/libdint_wl.so     workload clients (CPU C++: the reference's closed-loop clients restated)
  dint_b200/lib/dint_udp_server   the reference's UDP server front-end over the C ABI (recvmmsg / sendmmsg)
"""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
# DINT_LIB_TAG=<tag> (development only): load libdint_b200_<tag>.so, or build it with DINT_NVCC_DEFINES when it is missing
_TAG = os.environ.get("DINT_LIB_TAG", "")
LIB = os.path.join(LIBDIR, f"libdint_b200_{_TAG}.so" if _TAG else "libdint_b200.so")
WL_LIB = os.path.join(LIBDIR, "libdint_wl.so")
UDP_SERVER = os.path.join(LIBDIR, "dint_udp_server")

NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "-shared"]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _sources(exts):
    out = []
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in sorted(os.listdir(root)):
            if f.endswith(exts):
                out.append(os.path.join(root, f))
    return out


def find_nvcc():
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else None


def build(force=False, verbose=False):
    if not force and os.path.isdir(LIBDIR) and not os.access(LIBDIR, os.W_OK) and \
            all(os.path.exists(p) for p in (LIB, WL_LIB, UDP_SERVER)):
        return LIB                    # a read-only tree: use the libraries it was built with
    os.makedirs(LIBDIR, exist_ok=True)
    headers = _sources((".cuh", ".h"))
    units = _sources((".cu",))
    # a tagged library that exists is used as built: it may be a frozen build of another commit for an A/B run
    if (force or _newer(LIB, units + headers)) and not (_TAG and os.path.exists(LIB)):
        nvcc = find_nvcc()
        if nvcc is None:
            raise RuntimeError("nvcc not found: cannot build libdint_b200.so (there is no CPU fallback)")
        # DINT_NVCC_DEFINES: extra -D flags for A/B builds of a development variant (none exist at the moment)
        flags = [f for f in NVCC_FLAGS if f != "-shared"] + os.environ.get("DINT_NVCC_DEFINES", "").split() + \
            (["-Xptxas", "-v"] if verbose else [])
        # one object per unit (each kernel is compiled in exactly one), compiled in parallel; an object is rebuilt when
        # its unit or any header is newer.  Tagged builds keep tagged objects.
        objs, jobs = [], []
        for src in units:
            obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + (f"_{_TAG}" if _TAG else "") + ".o")
            objs.append(obj)
            if force or _newer(obj, [src] + headers):
                jobs.append((subprocess.Popen([nvcc] + flags + ["-c", "-o", obj, src]), obj))
        failed = [obj for proc, obj in jobs if proc.wait() != 0]
        for obj in failed:
            if os.path.exists(obj):
                os.remove(obj)
        if failed:
            raise RuntimeError("nvcc failed: " + ", ".join(os.path.basename(o) for o in failed))
        subprocess.run([nvcc] + NVCC_FLAGS + ["-o", LIB] + objs, check=True)
    wl_src = [os.path.join(CSRC, "workloads.cc"), os.path.join(CSRC, "txn_workloads.cc")]
    if os.path.exists(wl_src[0]) and (force or _newer(WL_LIB, wl_src + _sources((".h", ".cuh")))):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", WL_LIB] + wl_src, check=True)
    srv_src = os.path.join(CSRC, "udp_server.cc")
    if os.path.exists(srv_src) and (force or _newer(UDP_SERVER, [srv_src, LIB] + _sources((".h",)))):
        subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-o", UDP_SERVER, srv_src, "-L" + LIBDIR, "-ldint_b200",
                        "-Wl,-rpath,$ORIGIN", "-lpthread"], check=True)
    return LIB
