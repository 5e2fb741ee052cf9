// varlena.cuh -- what ORDER_SELS (order.cu) and PACK_STR_KEYS (colops.cu) both need to know about key columns: the varlena types, the storage
// size of every fixed-width key type, and the one check of varlena cells -- the lowest row whose cell points outside its area and the longest
// value of every column, measured on the device and read back as one record.
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

struct VarlenaStat {
    unsigned long long bad_inv[MO_ORDER_MAX_KEYS];   // ~(lowest row whose cell points outside the area), 0 = none
    unsigned maxlen[MO_ORDER_MAX_KEYS];              // longest non-NULL value
};

// enqueues the check of column k (rows [0, n), NULL rows skipped) into vs, which the caller zeroes first (order.cu)
int varlena_stat(ThreadCtx &t, const uint8_t *cells, const uint64_t *nulls, const uint8_t *area, uint64_t area_sz, uint64_t n, VarlenaStat *vs, int k);
// MO_RC_INVALID_ARGUMENT with the error "<what> k row r: ..." for the first of columns 0..ncols-1 with a bad cell or a value longer than
// MO_ORDER_MAX_VARLENA bytes; MO_RC_SUCCESS when there is none
int varlena_stat_error(const VarlenaStat &vs, int ncols, const char *what);

}  // namespace mob
