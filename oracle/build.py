"""Build the CPU oracle libraries (TEST INFRASTRUCTURE ONLY -- never imported by matrixone_b200/).

  oracle/liboracle_go.so      C restatement of the reference's Go batch loops (oracle_go.c), compiled the way
                              Go executes floating point: no -ffast-math, no FMA contraction.
  oracle/_ref/libmo_ref.so    the reference's own C kernels, compiled UNCHANGED from where they lie under
                              /root/reference/cgo with the reference's flags (cgo/Makefile:6-13).  Only built
                              when /root/reference exists (this container); the GPU box uses the prebuilt file.
  oracle/_ref/libusearch_ref.so  usearch 2.23.0 C API (exact search) from the vendored tarball
                              /root/reference/thirdparties/usearch-2.23.0.tar.gz, flags per
                              thirdparties/Makefile:60-90 (OpenMP on, SimSIMD off, fp16lib on).

  oracle/_ref/libbloom_ref.so the reference's bloom filter (cgo/bloom.c unchanged) + the xxHash 0.8.3 tarball it pins.
  oracle/libxxh3_host.so      matrixone_b200/csrc/xxh3_128.cuh compiled for the host (test-only wrapper xxh3_host.cpp).

No reference source is copied into the repo: tarballs are unpacked into a temp dir that is removed.
"""
import os
import shutil
import subprocess
import sys
import tarfile
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
REF_DIR = os.path.join(HERE, "_ref")


def _run(cmd, **kw):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, **kw)
    if r.returncode != 0:
        raise RuntimeError("command failed: %s\n%s" % (" ".join(cmd), r.stdout))
    return r.stdout


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources if os.path.exists(s))


def build_oracle_go(force=False):
    src = os.path.join(HERE, "oracle_go.c")
    out = os.path.join(HERE, "liboracle_go.so")
    if force or _newer(out, [src]):
        _run(["gcc", "-std=gnu11", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-shared", "-Wall",
              "-o", out, src, "-lm", "-lpthread"])
    return out


def build_mo_ref(force=False):
    """reference cgo C kernels, unchanged, reference flags."""
    out = os.path.join(REF_DIR, "libmo_ref.so")
    cgo = os.path.join(REF, "cgo")
    if not os.path.isdir(cgo):
        return out if os.path.exists(out) else None
    srcs = [os.path.join(cgo, f) for f in ("mo.c", "arith.c", "compare.c", "logic.c", "xcall.c")]
    if force or _newer(out, srcs):
        os.makedirs(REF_DIR, exist_ok=True)
        _run(["gcc", "-std=c99", "-g", "-O3", "-ffast-math", "-ftree-vectorize", "-funroll-loops", "-march=haswell",
              "-Wall", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-o", out] + srcs + ["-lm"])
    return out


def build_usearch_ref(force=False):
    out = os.path.join(REF_DIR, "libusearch_ref.so")
    tp = os.path.join(REF, "thirdparties")
    tarballs = [os.path.join(tp, f) for f in ("usearch-2.23.0.tar.gz", "fp16.tar.gz", "SimSIMD-6.5.3.tar.gz")]
    if not all(os.path.exists(t) for t in tarballs):
        return out if os.path.exists(out) else None
    if not (force or _newer(out, tarballs)):
        return out
    os.makedirs(REF_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="mo_b200_usearch_")
    try:
        for t in tarballs:
            with tarfile.open(t) as tf:
                tf.extractall(tmp)
        names = os.listdir(tmp)
        us = os.path.join(tmp, [n for n in names if n.lower().startswith("usearch")][0])
        fp16 = os.path.join(tmp, [n for n in names if n.lower().startswith("fp16")][0])
        simsimd = os.path.join(tmp, [n for n in names if n.lower().startswith("simsimd")][0])
        _run(["g++", "-std=c++17", "-O3", "-fPIC", "-shared", "-fopenmp", "-Wl,-Bsymbolic",
              "-DUSEARCH_USE_FP16LIB=1", "-DUSEARCH_USE_SIMSIMD=0", "-DUSEARCH_USE_OPENMP=1",
              "-I", os.path.join(us, "include"), "-I", os.path.join(us, "c"),
              "-I", os.path.join(fp16, "include"), "-I", os.path.join(simsimd, "include"),
              "-o", out, os.path.join(us, "c", "lib.cpp")])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return out


def build_mocl_ref(force=False):
    """the reference's own CUDA kernels (cgo/cuda/mocl.cu:4-92: l2distance_f32/_f64[_const], one thread per row), compiled UNCHANGED for sm_90a into a
    cubin.  The reference ships them as mocl_kernel64.fatbin loaded with cuModuleLoad (cgo/cuda/cuda.cpp:82-95); tools/ref_cuda_compare.py loads
    this cubin the same way and times the kernels next to ours (SURVEY.md section 2.3 bar (ii))."""
    out = os.path.join(REF_DIR, "mocl_sm90a.cubin")
    src = os.path.join(REF, "cgo", "cuda", "mocl.cu")
    if not os.path.exists(src):
        return out if os.path.exists(out) else None
    if force or _newer(out, [src]):
        os.makedirs(REF_DIR, exist_ok=True)
        _run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-cubin", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-o", out, src])
    return out


def build_bloom_ref(force=False):
    """the reference's bloom filter (cgo/bloom.c, UNCHANGED) with the xxHash 0.8.3 it pins (thirdparties/Makefile:26,45-49: xxhash.h copied
    next to it, XXH_INLINE_ALL).  Validates matrixone_b200/csrc/xxh3_128.cuh and bloom.cu."""
    out = os.path.join(REF_DIR, "libbloom_ref.so")
    src = os.path.join(REF, "cgo", "bloom.c")
    tarball = os.path.join(REF, "thirdparties", "xxHash-0.8.3.tar.gz")
    if not (os.path.exists(src) and os.path.exists(tarball)):
        return out if os.path.exists(out) else None
    if not (force or _newer(out, [src, tarball, os.path.join(HERE, "xxh3_ref_shim.c")])):
        return out
    os.makedirs(REF_DIR, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="mo_b200_xxhash_")
    try:
        with tarfile.open(tarball) as tf:
            tf.extractall(tmp)
        xx = os.path.join(tmp, [n for n in os.listdir(tmp) if n.lower().startswith("xxhash")][0])
        _run(["gcc", "-std=gnu11", "-O3", "-Wall", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-I", xx, "-I", os.path.join(REF, "cgo"), "-o", out, src, os.path.join(HERE, "xxh3_ref_shim.c"), "-lm"])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return out


def build_xxh3_host(force=False):
    """the device hash header compiled for the HOST (g++), so that the restatement can be pinned to the real xxHash without a GPU"""
    out = os.path.join(HERE, "libxxh3_host.so")
    hdr = os.path.join(os.path.dirname(HERE), "matrixone_b200", "csrc", "xxh3_128.cuh")
    src = os.path.join(HERE, "xxh3_host.cpp")
    if force or _newer(out, [hdr, src]):
        _run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-x", "c++", "-I", os.path.dirname(hdr), "-o", out, src])
    return out


def build_all(force=False, verbose=False):
    res = {"oracle_go": build_oracle_go(force), "xxh3_host": build_xxh3_host(force)}
    for name, fn in (("mo_ref", build_mo_ref), ("usearch_ref", build_usearch_ref), ("mocl_ref", build_mocl_ref), ("bloom_ref", build_bloom_ref)):
        try:
            res[name] = fn(force)
        except Exception as e:  # the reference libs are optional strengthening, the restatement is not
            res[name] = None
            if verbose:
                print("oracle/_ref %s not built: %s" % (name, e), file=sys.stderr)
    return res


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose=True))
