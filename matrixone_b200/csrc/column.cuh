// column.cuh -- input columns as every call reads them: the one rule for a 24-byte varlena cell, how an argument (a column or a const) is
// staged into an Operand, the key types of ORDER_SELS (order.cu) and PACK_STR_KEYS (colops.cu), and their one check of varlena cells -- the
// lowest row whose cell points outside its area and the longest value of every column, measured on the device and read back as one record.
#pragma once
#include "common.cuh"

namespace mob {

inline bool is_varlena(int T) {
    switch (T) {
    case MO_T_CHAR: case MO_T_VARCHAR: case MO_T_BINARY: case MO_T_VARBINARY: case MO_T_BLOB: case MO_T_TEXT: case MO_T_DATALINK: return true;
    }
    return false;
}

// storage bytes of a fixed-width key type (the key types of ORDER_SELS), 0 for any other type
inline int key_type_size(int T) {
    switch (T) {
    case MO_T_DECIMAL64: case MO_T_BIT: return 8;
    case MO_T_YEAR: case MO_T_ENUM: return 2;
    case MO_T_DECIMAL128: case MO_T_UUID: return 16;
    }
    return type_size(T);
}
// bytes per row of a key column: a varlena key's cells, or key_type_size; 0 for a type no key may have
inline int key_elem_size(int T) { return is_varlena(T) ? MO_VARLENA_SZ : key_type_size(T); }

// ---- the varlena cell, cgo/xcall.h:47-61 (== pkg/container/types/bytes.go:61-115): bs[0] <= 23 inline (the value is bs[1 .. 1 + bs[0])),
// else u32[1] = offset into the area and u32[2] = length.  w0, w1, w2 are the cell's first three 4-byte words, as the caller loaded them.
// ok = false when a non-inline cell has no area or points outside [0, area_sz).
struct VarlenaCell { uint32_t off, len; bool inl, ok; };
__host__ __device__ __forceinline__ VarlenaCell varlena_cell(uint32_t w0, uint32_t w1, uint32_t w2, const uint8_t *area, uint64_t area_sz) {
    const uint32_t b0 = w0 & 0xffu;
    if (b0 <= MO_VARLENA_INLINE_SZ) return VarlenaCell{0, b0, true, true};
    return VarlenaCell{w1, w2, false, area && (uint64_t)w1 + w2 <= area_sz};
}

// ---- operands
// the one const rule: a one-element vector is a const when len > 1; with len == 1 it is a column (both read element 0)
inline bool is_const(const mo_xcall_args_t &a, size_t elem, uint64_t len) { return a.dataSz == elem && len > 1; }

// a staged operand: data (and a varlena operand's area) and nulls in device memory
struct Operand {
    const void *data = nullptr;
    const uint64_t *nulls = nullptr;
    int cst = 0;                        // a const operand: every row reads element 0
    const uint8_t *area = nullptr;
    uint64_t area_sz = 0;
    const uint64_t *col_nulls() const { return cst ? nullptr : nulls; }   // the bitmap the null merge ORs in
    const uint64_t *cnull() const { return cst ? nulls : nullptr; }       // a const operand's null word, where a kernel can read it
};

// stages `rows` elements of args[k] of `what` (elem bytes per row: sizeof(T), 8, 16, or 24 for varlena cells, whose area is staged too)
inline int stage_rows(Stager &st, const mo_xcall_args_t &a, size_t elem, uint64_t rows, const char *what, int k, Operand &o) {
    if (!a.pdata || a.dataSz < elem * rows) {
        set_error("%s: operand %d holds %llu bytes, %llu needed", what, k, (unsigned long long)a.dataSz, (unsigned long long)(elem * rows));
        return MO_RC_INVALID_ARGUMENT;
    }
    o.data = st.in(a.pdata, elem * rows);
    o.nulls = (const uint64_t *)st.in(a.pnulls, a.pnulls ? ((rows + 63) / 64) * 8 : 0);
    if (elem == MO_VARLENA_SZ && a.parea && a.areaSz) { o.area = (const uint8_t *)st.in(a.parea, a.areaSz); o.area_sz = a.areaSz; }
    return st.failed ? MO_RC_INTERNAL_ERROR : MO_RC_SUCCESS;
}
// stages the operand args[k] of a len-row call: a const one is one element
inline int stage_operand(Stager &st, const mo_xcall_args_t &a, size_t elem, uint64_t len, const char *what, int k, Operand &o) {
    o = Operand{};
    o.cst = is_const(a, elem, len);
    return stage_rows(st, a, elem, o.cst ? 1 : len, what, k, o);
}

#ifdef __CUDACC__
// varlena cell i of cells, read byte by byte (any alignment): ptr = the value (inside the cell when inline)
struct VarlenaRef { const uint8_t *ptr; uint32_t len; bool ok, inl; };
__device__ __forceinline__ VarlenaRef varlena_ref(const uint8_t *cells, uint64_t i, const uint8_t *area, uint64_t areaSz) {
    const uint8_t *c = cells + 24 * i;
    uint32_t off, len;
    memcpy(&off, c + 4, 4); memcpy(&len, c + 8, 4);
    const VarlenaCell v = varlena_cell(c[0], off, len, area, areaSz);
    return VarlenaRef{v.inl ? c + 1 : area + v.off, v.len, v.ok, v.inl};
}

// A value of a varlena Operand.  An inline one (<= 23 bytes) stays in the three registers of its cell load; a long one is read from the area.
struct Str {
    uint64_t w0, w1, w2;
    const uint8_t *p;
    uint32_t len;
    bool inl;
    __device__ __forceinline__ uint32_t at(uint32_t j) const {
        if (inl) {
            const uint32_t k = j + 1;
            const uint64_t w = k < 8 ? w0 : (k < 16 ? w1 : w2);
            return (uint32_t)(w >> (8 * (k & 7))) & 0xffu;
        }
        return __ldg(p + j);
    }
};

// row `row` of c as three 8-byte loads (bytes when c.data is not 8-byte aligned); false: the cell is bad
__device__ __forceinline__ bool load_str(const Operand &c, uint64_t row, Str &s) {
    const uint8_t *cell = (const uint8_t *)c.data + 24 * (c.cst ? 0 : row);
    if ((reinterpret_cast<uintptr_t>(c.data) & 7) == 0) {
        const uint64_t *q = reinterpret_cast<const uint64_t *>(cell);
        s.w0 = __ldg(q); s.w1 = __ldg(q + 1); s.w2 = __ldg(q + 2);
    } else {
        s.w0 = s.w1 = s.w2 = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            s.w0 |= (uint64_t)__ldg(cell + k) << (8 * k);
            s.w1 |= (uint64_t)__ldg(cell + 8 + k) << (8 * k);
            s.w2 |= (uint64_t)__ldg(cell + 16 + k) << (8 * k);
        }
    }
    const VarlenaCell v = varlena_cell((uint32_t)s.w0, (uint32_t)(s.w0 >> 32), (uint32_t)s.w1, c.area, c.area_sz);
    s.inl = v.inl; s.len = v.len; s.p = v.inl ? nullptr : c.area + v.off;
    return v.ok;
}
#endif

// ---- key columns: ORDER_SELS and PACK_STR_KEYS
struct VarlenaStat {
    unsigned long long bad_inv[MO_ORDER_MAX_KEYS];   // ~(lowest row whose cell points outside the area), 0 = none
    unsigned maxlen[MO_ORDER_MAX_KEYS];              // longest non-NULL value
};

// enqueues the check of every varlena column k < n (by type[k]; rows [0, len), a const one its one row, NULL rows skipped) into vs, which
// the caller zeroes first: one launch per varlena column
int varlena_stats(ThreadCtx &t, const Operand *col, const int *type, int n, uint64_t len, VarlenaStat *vs);
// MO_RC_INVALID_ARGUMENT with the error "<what> k row r: ..." for the first of columns 0..ncols-1 with a bad cell or a value longer than
// MO_ORDER_MAX_VARLENA bytes; MO_RC_SUCCESS when there is none
int varlena_stat_error(const VarlenaStat &vs, int ncols, const char *what);

}  // namespace mob
