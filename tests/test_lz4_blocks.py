"""The LZ4 block writer and model of tests/lz4_blocks.py, checked against liblz4 (pyarrow lz4_raw) and the oracle decoder
(og_lz4_decode_block), and the coverage of csrc/lz4.cu's branches that its edge corpus reaches.  No GPU."""
import numpy as np
import pyarrow as pa

import lz4_blocks as L
import oracle_lib as O
from test_oracle_lz4 import corpus


def oracle_decode(block, dl):
    """(og_lz4_decode_block's return value, the bytes it wrote)"""
    src = np.frombuffer(block, np.uint8) if block else np.zeros(1, np.uint8)
    dst = np.zeros(max(dl, 1), np.uint8)
    n = O.go().og_lz4_decode_block(O.p(src), len(block), O.p(dst), dl)
    return n, dst[:max(n, 0)].tobytes()


def liblz4_decode(block, dl):
    """liblz4's decoded bytes, or None when it rejects the block"""
    try:
        return pa.decompress(block, decompressed_size=dl, codec="lz4_raw", asbytes=True)
    except (OSError, pa.ArrowException):
        return None


def test_written_blocks_decode_to_the_model_in_liblz4_and_the_oracle():
    blocks = [(s, t) for s, t in L.edge_table().values() if L.conformant(s, t)] + L.random_edge_corpus(3000)
    for seqs, tail in blocks:
        assert L.conformant(seqs, tail)
        blk, want = L.encode(seqs, tail), L.model(seqs, tail)
        assert liblz4_decode(blk, len(want)) == want
        assert oracle_decode(blk, len(want)) == (len(want), want)
        assert L.parse(blk)[:2] == (seqs, tail)


def test_parser_reads_liblz4_output_back_to_the_raw_bytes():
    for raw in corpus():
        comp = pa.compress(raw, codec="lz4_raw", asbytes=True)
        seqs, tail, _ = L.parse(comp)
        assert tail is not None and L.model(seqs, tail) == raw


def test_extension_bytes_are_written_as_the_format_says():
    assert L.encode([], b"x" * 15) == b"\xf0\x00" + b"x" * 15                         # nibble 15, extension 0
    assert L.encode([(b"ab", 2, 19)], b"") == b"\x2f" + b"ab" + b"\x02\x00" + b"\x00" + b"\x00"
    assert L.encode([], b"y" * 270)[:3] == b"\xf0\xff\x00"                            # 15 + 255 + 0
    assert L.encode([(b"a", 1, 4 + 15 + 255)], None) == b"\x1f" + b"a" + b"\x01\x00" + b"\xff\x00"
    assert L.model([(b"abc", 2, 5)], b"!") == b"abc" + b"bcbcb" + b"!"


def test_non_conformant_blocks_are_accepted_by_the_oracle_and_rejected_by_liblz4():
    """The LZ4 block format requires the last sequence to be literals only, its last 5 bytes to be literals and the last match to start 12
    or more bytes before the end; liblz4 rejects blocks that break these rules.  The oracle decoder (the restatement of the reference's
    Go decoder, which the device kernel follows) checks only what it needs to decode safely: every length and offset inside its buffers and
    the decoded size.  So it, and the GPU, accept these blocks and decode them by the sequence rules alone.  That is deliberate: the end rules
    exist for liblz4's fast copy loops, the decoded bytes are well defined without them, and every block a compressor writes is conformant.
    This test pins the difference so that it cannot change unnoticed."""
    rng = np.random.default_rng(7)
    nc = [(s, t) for name, (s, t) in L.edge_table().items() if name.startswith("nc_")]
    while len(nc) < 200:
        seqs, tail = L.random_edge_block(rng, conform=False, max_out=1 << 14)
        if rng.random() < 0.5:
            tail = None
        if not L.conformant(seqs, tail):
            nc.append((seqs, tail))
    ends_in_match = [(b"abcd", 4, 8)]
    assert L.encode(ends_in_match, None) == b"\x44abcd\x04\x00" and L.model(ends_in_match, None) == b"abcdabcdabcd"
    for seqs, tail in nc:
        assert not L.conformant(seqs, tail)
        blk, want = L.encode(seqs, tail), L.model(seqs, tail)
        assert oracle_decode(blk, len(want)) == (len(want), want)
        assert liblz4_decode(blk, len(want)) is None


def test_edge_corpus_reaches_every_kernel_branch():
    """the blocks the GPU exactness test decodes, at the misalignments it places them at, take every branch classify() names"""
    hit = set()
    for _, seqs, tail, mis in L.placed_corpus():
        hit |= L.classify(seqs, mis, tail)
    assert hit == L.BRANCHES, "branches no block reaches: %s" % sorted(L.BRANCHES - hit)


def test_classify_names_the_paths_of_hand_built_blocks():
    t = L.edge_table()
    assert {"match_ring_overlap", "ring_edge", "sync_taken"} <= L.classify(t["ring_edge_off3"][0], 0, t["ring_edge_off3"][1])
    assert {"match_far_overlap", "far_edge"} <= L.classify(t["far_edge_off3"][0], 0, t["far_edge_off3"][1])
    assert "sync_at_boundary" in L.classify(t["sync_boundary_off1000"][0], 0, t["sync_boundary_off1000"][1])
    assert "sync_past_boundary" in L.classify(t["sync_past_boundary_off1000"][0], 0, t["sync_past_boundary_off1000"][1])
    assert "first_fill_negative_base" not in L.classify([], 0, b"abc") and "first_fill_negative_base" in L.classify([], 5, b"abc")
