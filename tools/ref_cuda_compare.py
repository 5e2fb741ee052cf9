"""Kernel-vs-kernel: the reference's OWN CUDA kernels (cgo/cuda/mocl.cu, compiled unchanged by oracle/build.py into oracle/_ref/mocl_sm90a.cubin)
against this library's row-distance kernel, both on RESIDENT data (the reference's shim additionally allocates + copies per call, cuda.cpp:123-201;
that cost is not charged here).  2 M rows x 768-d f32, one side constant and both sides per-row; device time by CUDA events.

    python tools/ref_cuda_compare.py > ref_cuda_compare.json
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cuda.bindings import driver as cu  # noqa: E402

from matrixone_b200 import capi  # noqa: E402
from matrixone_b200.vector import DeviceBuffer, Vector  # noqa: E402


def ck(res):
    err = res[0]
    if int(err) != 0:
        raise RuntimeError("CUDA driver error %s" % err)
    return res[1] if len(res) == 2 else res[1:]


def main():
    n, dim = int(os.environ.get("ROWS", 2_000_000)), 768
    lib = capi.load_library()
    capi.check(lib.MoB200_Init(0), lib)
    ck(cu.cuInit(0))
    dev = ck(cu.cuDeviceGet(0))
    ctx = ck(cu.cuDevicePrimaryCtxRetain(dev))          # the runtime's primary context: the library's device pointers are valid in it
    ck(cu.cuCtxSetCurrent(ctx))
    cubin = open(os.path.join(ROOT, "oracle", "_ref", "mocl_sm90a.cubin"), "rb").read()
    mod = ck(cu.cuModuleLoadData(cubin))
    f_const = ck(cu.cuModuleGetFunction(mod, b"l2distance_f32_const"))
    f_vv = ck(cu.cuModuleGetFunction(mod, b"l2distance_f32"))
    # data: MatrixOne layout -- 24-byte varlena cells {0xffffffff, offset, len} + area
    A = DeviceBuffer(4 * n * dim, lib); B = DeviceBuffer(4 * n * dim, lib)
    capi.check(lib.MoB200_GenVectorsF32(20, 0, n, dim, A.ptr, None, 0, 1.0), lib)
    capi.check(lib.MoB200_GenVectorsF32(21, 0, n, dim, B.ptr, None, 0, 1.0), lib)
    cells = np.zeros((n, 6), dtype=np.uint32); cells[:, 0] = 0xFFFFFFFF; cells[:, 1] = (np.arange(n, dtype=np.uint64) * (4 * dim)).astype(np.uint32); cells[:, 2] = 4 * dim
    dcells = DeviceBuffer.from_numpy(cells.reshape(-1), lib)
    res_ref = DeviceBuffer(8 * n, lib); res_ours = DeviceBuffer(8 * n, lib)
    q = B.view(4 * dim)                                    # the constant operand: row 0 of B
    e0, e1 = ck(cu.cuEventCreate(0)), ck(cu.cuEventCreate(0))
    out = {"rows": n, "dim": dim, "what": "squared L2 (l2_distance_sq_xc), float diff / double accumulation (cgo/xcall.c semantics)"}

    def time_ref(fn, args, types, reps=5):
        best = []
        for _ in range(reps + 1):
            ck(cu.cuEventRecord(e0, 0))
            ck(cu.cuLaunchKernel(fn, (n + 255) // 256, 1, 1, 256, 1, 1, 0, 0, (tuple(args), tuple(types)), 0))      # CUDA_THREADS_PER_BLOCK 256, cuda.cpp:36
            ck(cu.cuEventRecord(e1, 0))
            ck(cu.cuEventSynchronize(e1))
            best.append(ck(cu.cuEventElapsedTime(e0, e1)))
        return float(np.median(best[1:]))

    def time_ours(vecs, reps=5):
        arr = (capi.XCallArgs * len(vecs))()
        for i, v in enumerate(vecs):
            arr[i] = v.fill_raw_ptr_len()
        err = (C.c_uint8 * 256)(); kms = C.c_float(); ts = []
        for _ in range(reps + 1):
            rc = lib.XCall(1, capi.XCALL_L2DISTANCE_SQ_F32, err, C.cast(arr, C.c_void_p), n)
            assert rc == 0, bytes(err[1:1 + err[0]])
            capi.check(lib.MoB200_LastKernelMs(C.byref(kms)), lib); ts.append(kms.value)
        return float(np.median(ts[1:]))

    cellv = lambda area: Vector(data_ptr=dcells.ptr, data_nbytes=24 * n, area_ptr=area.ptr, area_nbytes=4 * n * dim, length=n)
    resv = Vector(data_ptr=res_ours.ptr, data_nbytes=8 * n, length=n)
    for name, fn, bytes_moved in (("const", f_const, 4.0 * n * dim), ("vec_vec", f_vv, 8.0 * n * dim)):
        if name == "const":
            ms_ref = time_ref(fn, [res_ref.ptr, n, 4 * dim, True, dcells.ptr, A.ptr, q.ptr], [C.c_void_p, C.c_int, C.c_int, C.c_bool, C.c_void_p, C.c_void_p, C.c_void_p])
            qcell = np.zeros(6, dtype=np.uint32); qcell[0] = 0xFFFFFFFF; qcell[2] = 4 * dim
            dq = DeviceBuffer.from_numpy(qcell, lib)
            ms_ours = time_ours([resv, cellv(A), Vector(data_ptr=dq.ptr, data_nbytes=24, area_ptr=q.ptr, area_nbytes=4 * dim, length=n, const=True)])
        else:
            ms_ref = time_ref(fn, [res_ref.ptr, n, 4 * dim, True, dcells.ptr, A.ptr, dcells.ptr, B.ptr], [C.c_void_p, C.c_int, C.c_int, C.c_bool, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p])
            ms_ours = time_ours([resv, cellv(A), cellv(B)])
        r_ref = res_ref.to_numpy(np.float64); r_ours = res_ours.to_numpy(np.float64)
        out[name] = {"reference_mocl_ms": ms_ref, "ours_ms": ms_ours, "speedup": ms_ref / ms_ours, "reference_gbs": bytes_moved / ms_ref / 1e6, "ours_gbs": bytes_moved / ms_ours / 1e6,
                     "max_rel_diff": float(np.max(np.abs(r_ref - r_ours) / np.maximum(np.abs(r_ref), 1e-30))), "identical": bool(np.array_equal(r_ref, r_ours))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
