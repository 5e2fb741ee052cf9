"""Sequence-level LZ4 block writer, plain decoded-bytes model and branch classifier for the block decode tests (no GPU).

A block is written from explicit sequences (literals, offset, match_len) plus the literals of the last sequence, following the published
LZ4 block format (lz4_Block_format.md): token = literal-length nibble << 4 | (match_len - 4) nibble, a nibble of 15 continued by extension
bytes that are 255 until the last one (which may be 0), the literals, a 2-byte little-endian offset, the match-length extension.  The end
of block rules of that format (the last sequence is literals only, its last 5 bytes are literals, the last match starts 12 or more bytes
before the end) hold for blocks written with `conformant` sequences; encode() writes the others too (tail=None: the block ends in a match),
because the decoders here accept them and the tests pin that.

`model` applies the sequences to an output buffer; `classify` replays the control flow of csrc/lz4.cu's decode loop (window refills, ring
or global match paths, the conditional sync) and names the branches a block takes, so a test can assert that its corpus reaches all of them.
"""
import struct

import numpy as np

# copied from csrc/lz4.cu (kWin, kRing): the per-warp source window and output ring sizes
KWIN = 512
KRING = 4096

BRANCHES = frozenset([
    "first_fill_negative_base",                                  # the first window of a block whose source is not 16-byte aligned
    "refill_token", "refill_lit_ext", "refill_offset_lo", "refill_offset_hi", "refill_match_ext",   # W.byte() ran past the window
    "lit_refill",                                                # a literal run of <= KWIN - 16 bytes refilled into the window
    "lit_window", "lit_global",                                  # literal copy served from the window / from global memory
    "lit_wraps_ring",                                            # a literal run longer than the ring
    "match_ring", "match_ring_overlap", "match_far", "match_far_overlap",
    "ring_edge",                                                 # offset <= KRING, mlen == KRING - offset: the longest ring match
    "far_edge",                                                  # offset <= KRING, mlen == KRING - offset + 1: the shortest far one
    "sync_taken", "sync_skipped",
    "sync_at_boundary",                                          # offset + mlen + 2 * KWIN == KRING: skipped
    "sync_past_boundary",                                        # offset + mlen + 2 * KWIN == KRING + 1: taken
])


def _length(out, n):
    """the 255-terminated extension of a length whose nibble is 15 (n >= 15): 255 while 255 or more remain, then the rest (may be 0)"""
    n -= 15
    while n >= 255:
        out.append(255)
        n -= 255
    out.append(n)


def encode(seqs, tail_literals=b""):
    """A raw LZ4 block from [(literals, offset, match_len), ...] and the last sequence's literals.  tail_literals=None ends the block with
    the last match (not conformant; the decoders here accept it, liblz4 does not)."""
    out = bytearray()
    for lit, off, ml in seqs:
        assert 1 <= off <= 0xFFFF and ml >= 4
        ln, mn = len(lit), ml - 4
        out.append((min(ln, 15) << 4) | min(mn, 15))
        if ln >= 15:
            _length(out, ln)
        out += lit
        out += struct.pack("<H", off)
        if mn >= 15:
            _length(out, mn)
    if tail_literals is not None:
        ln = len(tail_literals)
        out.append(min(ln, 15) << 4)
        if ln >= 15:
            _length(out, ln)
        out += tail_literals
    return bytes(out)


def model(seqs, tail_literals=b""):
    """The decoded bytes: literals appended, then match byte i = output byte (position - offset + i).  For i >= offset that byte is match
    byte i - offset itself, so an overlapping match (offset < match_len) repeats the last `offset` bytes before it."""
    out = bytearray()
    for lit, off, ml in seqs:
        out += lit
        if not 1 <= off <= len(out):
            raise ValueError("offset %d before the start of the block (position %d)" % (off, len(out)))
        last = out[len(out) - off:]
        out += last[:ml] if off >= ml else (last * (ml // off + 1))[:ml]
    if tail_literals is not None:
        out += tail_literals
    return bytes(out)


def parse(block):
    """(seqs, tail_literals, control byte positions) of a raw block; tail_literals is None when the block ends in a match.  ValueError when
    the block is cut inside a sequence.  The control positions are the token, extension and offset bytes."""
    seqs, ctrl, ip, n = [], [], 0, len(block)

    def ext(v):
        nonlocal ip
        if v == 15:
            while True:
                if ip >= n:
                    raise ValueError("length extension past the end")
                ctrl.append(ip)
                e = block[ip]; ip += 1; v += e
                if e != 255:
                    break
        return v

    while ip < n:
        ctrl.append(ip)
        tok = block[ip]; ip += 1
        ln = ext(tok >> 4)
        if ip + ln > n:
            raise ValueError("literals past the end")
        lit = bytes(block[ip:ip + ln]); ip += ln
        if ip == n:
            return seqs, lit, ctrl
        if ip + 2 > n:
            raise ValueError("offset past the end")
        ctrl += [ip, ip + 1]
        off = block[ip] | block[ip + 1] << 8; ip += 2
        seqs.append((lit, off, ext(tok & 15) + 4))
    return seqs, None, ctrl


def conformant(seqs, tail_literals):
    """the end-of-block rules of the LZ4 block format (what liblz4's decoder enforces on top of the sequence syntax)"""
    if tail_literals is None:
        return False
    total = len(model(seqs, tail_literals))
    if not seqs:
        return True
    last_match = total - len(tail_literals) - seqs[-1][2]
    return len(tail_literals) >= 5 and last_match <= total - 12


def classify(seqs, src_misalignment=0, tail_literals=b""):
    """The branch names (BRANCHES) csrc/lz4.cu's decode loop takes on encode(seqs, tail_literals) placed at src_misalignment mod 16."""
    blk = encode(seqs, tail_literals)
    sl, m, hit = len(blk), src_misalignment % 16, set()
    fill = lambda ip: ip - (m + ip) % 16               # the window base: src + ip rounded down to 16 bytes, relative to src
    base = fill(0)
    if base < 0:
        hit.add("first_fill_negative_base")

    def byte(ip, where):
        nonlocal base
        if ip - base >= KWIN:
            base = fill(ip)
            hit.add("refill_" + where)
        return blk[ip]

    def ext(v, ip, where):
        if v == 15:
            while True:
                e = byte(ip, where); ip += 1; v += e
                if e != 255:
                    break
        return v, ip

    ip = op = 0
    while ip < sl:
        token = byte(ip, "token"); ip += 1
        lit, ip = ext(token >> 4, ip, "lit_ext")
        if lit:
            if ip + lit - base > KWIN and lit <= KWIN - 16:
                base = fill(ip)
                hit.add("lit_refill")
            hit.add("lit_window" if ip + lit - base <= KWIN else "lit_global")
            if lit > KRING:
                hit.add("lit_wraps_ring")
        ip += lit; op += lit
        if ip >= sl:
            break
        offset = byte(ip, "offset_lo") | byte(ip + 1, "offset_hi") << 8
        ip += 2
        mlen, ip = ext(token & 15, ip, "match_ext")
        mlen += 4
        ring = offset <= KRING and mlen <= KRING - offset
        hit.add(("match_ring" if ring else "match_far") + ("_overlap" if offset < mlen else ""))
        if offset <= KRING and mlen == KRING - offset:
            hit.add("ring_edge")
        if offset <= KRING and mlen == KRING - offset + 1:
            hit.add("far_edge")
        op += mlen
        edge = offset + mlen + 2 * KWIN
        hit.add("sync_taken" if edge > KRING else "sync_skipped")
        if edge == KRING:
            hit.add("sync_at_boundary")
        if edge == KRING + 1:
            hit.add("sync_past_boundary")
    return hit


# ------------------------------------------------------------------------------------------------------------- edge blocks
LIT_EDGES = [0, 1, 14, 15, 16, 269, 270, 271] + list(range(KWIN - 17, KWIN + 2)) + [KRING - 1, KRING, KRING + 1, 20000]
OFF_EDGES = [1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 31, 32, 33, 63, 64, 65, KRING - 1, KRING, KRING + 1, 8191, 65535]


def _match_edges(off):
    return [4, 5, 18, 19, 20, 273, 274, 275, 529, KRING - off - 1, KRING - off, KRING - off + 1, KRING, KRING + 1, 70000,
            KRING - 2 * KWIN - off, KRING - 2 * KWIN - off + 1]


def random_bytes(rng, n):
    """literal bytes: never one repeated value, so a match read from the wrong place shows up"""
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def random_edge_block(rng, conform=True, max_out=1 << 17):
    """(seqs, tail) drawn mostly from the edge values; every offset reaches inside the output (offset <= position)"""
    seqs, op = [], 0
    for _ in range(int(rng.integers(1, 6))):
        ln = int(rng.choice(LIT_EDGES)) if rng.random() < 0.8 else int(rng.integers(0, 600))
        if op + ln == 0:
            ln = 1
        if op + ln > max_out:
            break
        op += ln
        offs = [o for o in OFF_EDGES if o <= op]
        off = int(rng.choice(offs)) if offs and rng.random() < 0.85 else int(rng.integers(1, min(op, 0xFFFF) + 1))
        mls = [m for m in _match_edges(off) if m >= 4 and op + m <= max_out]
        ml = int(rng.choice(mls)) if mls and rng.random() < 0.85 else int(rng.integers(4, 300))
        seqs.append((random_bytes(rng, ln), off, ml))
        op += ml
    tl = int(rng.choice([0, 1, 5, 6, 12, 15, 16, 300]))
    if conform:
        tl = max(tl, 5, 12 - (seqs[-1][2] if seqs else 0))
    return seqs, random_bytes(rng, tl)


def random_edge_corpus(n, seed=0):
    rng = np.random.default_rng(seed)
    return [random_edge_block(rng) for _ in range(n)]


def edge_table():
    """Hand-placed blocks, {name: (seqs, tail)}; each is conformant unless its name says otherwise."""
    rng = np.random.default_rng(12345)
    b = lambda n: random_bytes(rng, n)
    t = {}
    t["literals_only_1"] = ([], b(1))
    t["literals_only_15_ext_0"] = ([], b(15))
    t["nibble15_ext0_both"] = ([(b(15), 7, 19)], b(15))
    t["ext_255_then_0"] = ([(b(270), 16, 274)], b(270))
    t["ext_255_255_then_0"] = ([(b(525), 64, 529)], b(20))
    for off in (1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 31, 32, 33, 63, 64, 65):
        t["ring_overlap_off%d" % off] = ([(b(max(off, 40)), off, 200)], b(12))
        if KRING - off >= 4:
            t["ring_edge_off%d" % off] = ([(b(max(off, 40)), off, KRING - off)], b(12))
        t["far_edge_off%d" % off] = ([(b(max(off, 40)), off, KRING - off + 1)], b(12))
        t["far_overlap_long_off%d" % off] = ([(b(max(off, 40)), off, 9000 + off)], b(12))
    for off in (KRING - 1, KRING, KRING + 1, 8191):
        t["far_off%d" % off] = ([(b(off + 100), off, 300), (b(3), off, 4)], b(12))
    t["ring_edge_off4092_len4"] = ([(b(KRING), KRING - 4, 4)], b(12))
    t["far_edge_off4091_len6"] = ([(b(KRING), KRING - 5, 6)], b(12))
    t["offset_65535_last"] = ([(b(65535), 65535, 300)], b(12))
    t["offset_65535_overlapping"] = ([(b(65535), 65535, 70000)], b(12))
    t["literal_wraps_ring"] = ([(b(KRING + 1), 33, 100), (b(20000), KRING, 40)], b(KRING - 1))
    t["long_match_then_long_literal"] = ([(b(64), 17, 70000), (b(KRING), 5, KRING + 1)], b(20))
    # the trailing sync: offset + mlen + 2 * KWIN at KRING (skipped) and at KRING + 1 (taken), then a full-window literal and a match
    for off in (1000, 31, 100):
        ml = KRING - 2 * KWIN - off
        t["sync_boundary_off%d" % off] = ([(b(max(off, 40)), off, ml), (b(KWIN - 16), 7, 50), (b(40), off, 64)], b(12))
        t["sync_past_boundary_off%d" % off] = ([(b(max(off, 40)), off, ml + 1), (b(KWIN - 16), 7, 50), (b(40), off, 64)], b(12))
    # the token stream walks across the first window's end at every position: the offset, extensions and next token straddle it
    for ln in range(480, 514):
        t["window_walk_%d" % ln] = ([(b(ln), 8, 539), (b(300), 16, 20), (b(15), 3, 4 + 15 + 255)], b(20))
    # not conformant (accepted by the decoders here, rejected by liblz4)
    t["nc_ends_in_match"] = ([(b"abcd", 4, 8)], None)
    t["nc_ends_in_long_match"] = ([(b(40), 3, 5000)], None)
    t["nc_match_in_last_5"] = ([(b(20), 4, 4)], b(2))
    t["nc_match_starts_late"] = ([(b(20), 20, 4)], b(5))
    return t


def placed_corpus(n_random=3000):
    """[(name, seqs, tail, source misalignment)]: every edge-table block at misalignments 0..15, random edge block i at i % 16"""
    out = [(name, s, tl, m) for name, (s, tl) in edge_table().items() for m in range(16)]
    out += [("random_%d" % i, s, tl, i % 16) for i, (s, tl) in enumerate(random_edge_corpus(n_random))]
    return out
