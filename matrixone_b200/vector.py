"""Host-side mirror of the reference containers that cross the cgo boundary, for the Python harness (tests, bench).

  Vector         <-> pkg/container/vector/vector.go:43-68 (data / area / nulls / const class) with
                     fill_raw_ptr_len() == Vector.FillRawPtrLen (vector.go:5161-5172)
  bitmap helpers <-> pkg/common/bitmap/bitmap.go (LSB-first uint64 words, set = NULL)
  varlena cells  <-> pkg/container/types/bytes.go:26-115 == cgo/varlena.h:63-105 (24-byte cell: bs[0] <= 23 inline,
                     else u32[1] = offset into area, u32[2] = length)
  xcall()        <-> XCallFunction.XCall + c_xcall (pkg/sql/plan/function/cxcall.go:65-172): result first, nulls
                     pre-OR-ed, 256-byte Pascal error string
  DeviceBuffer   <-> a resident column: device memory owned through MoB200_DeviceAlloc

Nothing here computes results: it only lays out bytes and calls the C-ABI.
"""
import ctypes as C

import numpy as np

from . import capi

VARLENA_SZ = 24
VARLENA_INLINE = 23


# ---------------------------------------------------------------------------------------------- bitmaps
def bitmap_words(nbits):
    return (nbits + 63) // 64


def bitmap_from_bools(mask):
    """mask[i] True => row i NULL.  Returns uint64 words (trailing bits zero, bitmap.go:27-31)."""
    mask = np.asarray(mask, dtype=bool)
    n = mask.shape[0]
    padded = np.zeros(bitmap_words(n) * 64, dtype=np.uint8)
    padded[:n] = mask
    return np.packbits(padded.reshape(-1, 8), axis=1, bitorder="little").reshape(-1).view(np.uint64).copy()


def bitmap_to_bools(words, nbits):
    words = np.ascontiguousarray(words, dtype=np.uint64)
    bits = np.unpackbits(words.view(np.uint8), bitorder="little")
    return bits[:nbits].astype(bool)


# ---------------------------------------------------------------------------------------------- varlena
def varlena_column(rows, dtype=np.float32):
    """Build (cells uint8[n*24], area uint8[]) for a list of 1-D arrays, MatrixOne layout."""
    n = len(rows)
    cells = np.zeros((n, VARLENA_SZ), dtype=np.uint8)
    chunks, off = [], 0
    for i, r in enumerate(rows):
        b = np.ascontiguousarray(r, dtype=dtype).view(np.uint8).reshape(-1)
        ln = b.shape[0]
        if ln <= VARLENA_INLINE:
            cells[i, 0] = ln
            cells[i, 1:1 + ln] = b
        else:
            u32 = cells[i].view(np.uint32)
            u32[0] = 0xFFFFFFFF
            u32[1] = off
            u32[2] = ln
            chunks.append(b)
            off += ln
    area = np.concatenate(chunks) if chunks else np.zeros(0, dtype=np.uint8)
    return cells.reshape(-1), area


def varlena_column_from_matrix(mat):
    """Fast path for a dense [n, dim] matrix whose rows are all 'big' (dim*itemsize > 23)."""
    mat = np.ascontiguousarray(mat)
    n, dim = mat.shape
    ln = dim * mat.itemsize
    assert ln > VARLENA_INLINE
    cells = np.zeros((n, 6), dtype=np.uint32)
    cells[:, 0] = 0xFFFFFFFF
    cells[:, 1] = (np.arange(n, dtype=np.uint64) * ln).astype(np.uint32)
    cells[:, 2] = ln
    return cells.view(np.uint8).reshape(-1), mat.view(np.uint8).reshape(-1)


def varlena_bytes_column(values):
    """Build (cells uint8[n*24], area uint8[]) for a list of bytes values (CHAR / VARCHAR / TEXT / BLOB ...), MatrixOne layout; the
    non-inline values go into the area in row order."""
    n = len(values)
    lens = np.fromiter((len(v) for v in values), dtype=np.int64, count=n)
    flat = np.frombuffer(b"".join(values), dtype=np.uint8)
    starts = np.cumsum(lens) - lens
    cells = np.zeros((n, VARLENA_SZ), dtype=np.uint8)
    inl = lens <= VARLENA_INLINE
    il = lens[inl]
    rows = np.repeat(np.flatnonzero(inl), il)
    j = np.arange(rows.size) - np.repeat(np.cumsum(il) - il, il)
    cells[rows, 1 + j] = flat[np.repeat(starts[inl], il) + j]
    cells[inl, 0] = il
    big = ~inl
    bl = lens[big]
    u32 = cells.view(np.uint32)
    u32[big, 0] = 0xFFFFFFFF
    u32[big, 1] = (np.cumsum(bl) - bl).astype(np.uint32)
    u32[big, 2] = bl.astype(np.uint32)
    area = flat[np.repeat(big, lens)] if bl.size else np.zeros(0, dtype=np.uint8)
    return cells.reshape(-1), np.ascontiguousarray(area)


def varlena_char1_column(chars):
    """char(1)/varchar(1) column (TPC-H l_returnflag / l_linestatus): every cell inline, len 1."""
    chars = np.asarray(chars, dtype=np.uint8)
    cells = np.zeros((chars.shape[0], VARLENA_SZ), dtype=np.uint8)
    cells[:, 0] = 1
    cells[:, 1] = chars
    return cells.reshape(-1)


# ---------------------------------------------------------------------------------------------- device memory
class DeviceBuffer:
    """A resident column / buffer in HBM."""

    def __init__(self, nbytes, lib=None):
        self.lib = lib or capi.load_library()
        self.nbytes = int(nbytes)
        p = C.c_void_p()
        capi.check(self.lib.MoB200_DeviceAlloc(max(self.nbytes, 1), C.byref(p)), self.lib)
        self.ptr = p.value

    @classmethod
    def from_numpy(cls, arr, lib=None):
        arr = np.ascontiguousarray(arr)
        b = cls(arr.nbytes, lib)
        if arr.nbytes:
            capi.check(b.lib.MoB200_Upload(b.ptr, arr.ctypes.data, arr.nbytes), b.lib)
        return b

    def to_numpy(self, dtype, count=None):
        dt = np.dtype(dtype)
        count = self.nbytes // dt.itemsize if count is None else count
        out = np.empty(count, dtype=dt)
        if out.nbytes:
            capi.check(self.lib.MoB200_Download(out.ctypes.data, self.ptr, out.nbytes), self.lib)
        return out

    def view(self, nbytes, offset=0):
        """non-owning window [offset, offset + nbytes) of this buffer (a prefix / block range of a resident column)"""
        v = DeviceBuffer.__new__(DeviceBuffer)
        v.lib, v.nbytes, v.ptr, v.owner = self.lib, int(nbytes), self.ptr + int(offset), self
        return v

    def free(self):
        if self.ptr and getattr(self, "owner", None) is None:
            self.lib.MoB200_DeviceFree(self.ptr)
        self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class PinnedArray:
    """numpy view over pinned host memory from MoB200_HostAlloc (what MatrixOne's off-heap allocator would hand out)."""

    def __init__(self, shape, dtype, lib=None):
        self.lib = lib or capi.load_library()
        dt = np.dtype(dtype)
        n = int(np.prod(shape)) * dt.itemsize
        p = C.c_void_p()
        capi.check(self.lib.MoB200_HostAlloc(max(n, 1), C.byref(p)), self.lib)
        self.ptr = p.value
        buf = (C.c_uint8 * max(n, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=dt, count=int(np.prod(shape))).reshape(shape)

    def free(self):
        if self.ptr:
            self.array = None
            self.lib.MoB200_HostFree(self.ptr)
            self.ptr = None


# ---------------------------------------------------------------------------------------------- Vector
class Vector:
    """Minimal vector.Vector: data / nulls / area are host numpy buffers or DeviceBuffers, or raw device pointers (ptr + nbytes)."""

    def __init__(self, data=None, nulls=None, area=None, length=None, const=False,
                 data_ptr=None, data_nbytes=0, nulls_ptr=None, area_ptr=None, area_nbytes=0):
        self.data, self.nulls, self.area = data, nulls, area
        self.const = const
        self.length = length if length is not None else (0 if data is None else len(data))
        self.data_ptr, self.data_nbytes = data_ptr, data_nbytes
        self.nulls_ptr, self.area_ptr, self.area_nbytes = nulls_ptr, area_ptr, area_nbytes
        self._keep = []

    def _raw(self, x, dtype=None):
        """(address, bytes, buffer) of a DeviceBuffer, or of x as a contiguous host array kept alive with this Vector"""
        if isinstance(x, DeviceBuffer):
            return x.ptr, x.nbytes, x
        x = np.ascontiguousarray(x, dtype)
        self._keep.append(x)
        return x.ctypes.data, x.nbytes, x

    def fill_raw_ptr_len(self):
        """[pnulls, nbits, pdata, dataSz, parea, areaSz] -- Vector.FillRawPtrLen, vector.go:5161-5172.  An empty host area passes no
        pointer; a device area always passes its own."""
        a = capi.XCallArgs()
        if self.data_ptr is not None:
            a.pdata, a.dataSz = self.data_ptr, self.data_nbytes
        elif self.data is not None:
            a.pdata, a.dataSz, _ = self._raw(self.data)
        if self.nulls_ptr is not None:
            a.pnulls, a.nullCnt = self.nulls_ptr, self.length
        elif self.nulls is not None:
            a.pnulls, _, self.nulls = self._raw(self.nulls, np.uint64)
            a.nullCnt = self.length
        if self.area_ptr is not None:
            a.parea, a.areaSz = self.area_ptr, self.area_nbytes
        elif isinstance(self.area, DeviceBuffer) or (self.area is not None and len(self.area)):
            a.parea, a.areaSz, _ = self._raw(self.area)
        return a


def xcall(func_id, vectors, length, runtime_id=1, lib=None, raise_on_error=True):
    """XCallFunction.XCall (cxcall.go:102-172): vectors[0] is the result.  Returns (rc, error text)."""
    lib = lib or capi.load_library()
    arr = (capi.XCallArgs * len(vectors))()
    for i, v in enumerate(vectors):
        arr[i] = v.fill_raw_ptr_len() if isinstance(v, Vector) else v
    err = (C.c_uint8 * 256)()
    rc = lib.XCall(runtime_id, func_id, err, C.cast(arr, C.c_void_p), length)
    msg = bytes(err[1:1 + err[0]]).decode(errors="replace") if err[0] else ""
    if rc != 0 and raise_on_error:
        raise capi.MoError(rc, "xcall xfunc failed, error code %d, %s" % (rc, msg))
    return rc, msg


# ---------------------------------------------------------------------------------------------- marshalled vectors (object blocks)
def marshal_vector(oid, data, length, area=b"", nulls=None, size=None, width=0, scale=0, const=False, sorted_flag=False):
    """Vector.MarshalBinary (pkg/container/vector/vector.go:718-764) for the test harness: class, types.Type (16 bytes), length, dataLen + data,
    areaLen + area, nspLen + bitmap.Marshal (count, len, size, words; nothing when no row is NULL), sorted."""
    data = np.ascontiguousarray(data).view(np.uint8).reshape(-1).tobytes()
    area = bytes(area)
    out = bytearray()
    out += bytes([1 if const else 0])
    out += bytes([oid & 0xFF, 0, 0, 0]) + np.array([size if size is not None else (len(data) // max(length, 1)), width, scale], dtype=np.int32).tobytes()
    out += np.uint32(length).tobytes() + np.uint32(len(data)).tobytes() + data
    out += np.uint32(len(area)).tobytes() + area
    nsp = b""
    if nulls is not None:
        words = np.ascontiguousarray(nulls, dtype=np.uint64)
        cnt = int(sum(bin(int(w)).count("1") for w in words))
        if cnt:
            nsp = np.int64(cnt).tobytes() + np.uint64(length).tobytes() + np.uint64(words.nbytes).tobytes() + words.tobytes()
    out += np.uint32(len(nsp)).tobytes() + nsp
    out += bytes([1 if sorted_flag else 0])
    return bytes(out)
