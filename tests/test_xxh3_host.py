"""The device hash header (matrixone_b200/csrc/xxh3_128.cuh, compiled for the host by oracle/build.py) against the REAL xxHash 0.8.3 of the
tarball the reference pins (thirdparties/Makefile:26): every input-length class of XXH3_128bits_withSeed, several seeds, and the 8-byte
integer path cgo/bloom.c:31-37 uses.  The real hashes of these inputs are stored in tests/golden/xxh3_128_*_ref.npy (computed with
the reference's bloom.c + xxHash build, oracle/build.py build_bloom_ref).  No GPU needed."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


GOLDEN = os.path.join(ROOT, "tests", "golden")


def _mine():
    from oracle import build as oracle_build
    mine = C.CDLL(oracle_build.build_xxh3_host())
    mine.mob_xxh3_128_bytes.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]
    mine.mob_xxh3_128_u64.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p]
    return mine


def test_every_length_class_matches_real_xxhash():
    mine = _mine()
    want = np.load(os.path.join(GOLDEN, "xxh3_128_bytes_ref.npy"))
    rng = np.random.default_rng(1)
    buf = rng.integers(0, 256, 6000, dtype=np.uint8)
    b = np.zeros(2, np.uint64)
    for i, seed in enumerate((0, 1, 0x9E3779B185EBCA87, 0xFFFFFFFFFFFFFFFF, int(rng.integers(0, 2 ** 63)))):
        for j, n in enumerate(list(range(0, 1100)) + [2047, 2048, 2049, 4096, 5990]):
            mine.mob_xxh3_128_bytes(buf.ctypes.data + 3, n, seed, b.ctypes.data)   # + 3: unaligned input
            assert (want[i, j] == b).all(), (seed, n)


def test_integer_key_path_matches_real_xxhash():
    mine = _mine()
    want = iter(np.load(os.path.join(GOLDEN, "xxh3_128_u64_ref.npy")))
    rng = np.random.default_rng(2)
    b = np.zeros(2, np.uint64)
    for seed in (0, 7, 0xDEADBEEFCAFEF00D):
        for k in list(rng.integers(0, 2 ** 64, 500, dtype=np.uint64)) + [0, 1, 2 ** 64 - 1, 2 ** 63]:
            mine.mob_xxh3_128_u64(int(k), seed, b.ctypes.data)
            assert (next(want) == b).all(), (seed, k)
