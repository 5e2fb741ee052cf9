"""The 24-byte varlena cell edges that every reader of a cell shares (csrc/column.cuh, varlena_cell): a non-inline cell is good when
off + len <= areaSz, with the sum taken in 64 bits, and there is an area.  These helpers build the edge cells out of a column whose values
are all non-inline, and place cells at a device address with a chosen misalignment."""
import numpy as np

from matrixone_b200 import capi
from matrixone_b200.vector import DeviceBuffer, varlena_bytes_column

WRAP_OFF, WRAP_LEN = 0xFFFFFFF0, 0x20        # off + len wraps 32 bits to 0x10, inside any area


def set_cell(cells, row, off, ln):
    """row's cell becomes a non-inline cell (off, ln)"""
    u = cells.reshape(-1, 24)[row].view(np.uint32)
    u[0], u[1], u[2] = 0xFFFFFFFF, off, ln


def edges(values, end_row, past_row, wrap_row):
    """(cells, area) of values, every value non-inline, with end_row pointing at the area's last len(values[-1]) bytes (good: it ends at
    areaSz and reads values[-1]), past_row ending at areaSz + 1 and wrap_row at (0xFFFFFFF0, 0x20); a row given as None is left alone"""
    assert min(len(v) for v in values) > 23
    cells, area = varlena_bytes_column(values)
    cells = cells.copy()
    L = len(values[-1])
    if end_row is not None:
        set_cell(cells, end_row, area.size - L, L)
    if past_row is not None:
        set_cell(cells, past_row, area.size - L + 1, L)
    if wrap_row is not None:
        set_cell(cells, wrap_row, WRAP_OFF, WRAP_LEN)
    return cells, area


def on_device(arr, shift):
    """arr uploaded `shift` bytes past a 256-byte aligned allocation: (owner to free, view)"""
    arr = np.ascontiguousarray(arr)
    buf = DeviceBuffer(arr.nbytes + 16)
    v = buf.view(arr.nbytes, shift)
    capi.check(buf.lib.MoB200_Upload(v.ptr, arr.ctypes.data, arr.nbytes), buf.lib)
    return buf, v


SHIFTS = (8, 1)      # 8-byte but not 16-byte aligned, and 1-byte misaligned
