"""Host restatement of the reference's LIKE and string comparisons, for the tests of MO_XCALL_GO_LIKE and MO_XCALL_GO_COMPARE over varlena
operands.  Written from pkg/sql/plan/function/func_builtin_regexp.go and func_compare.go, and kept in step with them:

  like(s, pat, pat_const)  likeFn (:51-69): a const pattern goes through optimize_rule (optimizeRuleForLike, :91-280) first; a pattern the
                           rule declines, and every column pattern, through regular_match (regularMatchForLikeOp, :618-672).
  optimize_rule(pat)       None when the rule declines the pattern, else a function bytes -> bool.  Byte level: `_` is one byte.
  regular_match(pat, s)    ^(?s:...)$ over runes: the pattern's replace() written out as Python `re` over the decoded rune sequences.
  compare(op, a, b)        bytes.Equal / bytes.Compare, which Python's bytes operators are.

NULL handling and skipped rows are the callers' (the GO conventions of include/mo_b200.h).
"""
import re

RUNE_ERROR = 0xFFFD


def decode_rune(b, i):
    """utf8.DecodeRune(b[i:]) -> (rune, size): an invalid, overlong, surrogate or truncated sequence is (RuneError, 1)"""
    b0 = b[i]
    n = len(b) - i
    if b0 < 0x80:
        return b0, 1
    if b0 < 0xC2 or b0 > 0xF4:
        return RUNE_ERROR, 1
    sz = 2 if b0 < 0xE0 else (3 if b0 < 0xF0 else 4)
    if n < sz:
        return RUNE_ERROR, 1
    lo = {0xE0: 0xA0, 0xF0: 0x90}.get(b0, 0x80)
    hi = {0xED: 0x9F, 0xF4: 0x8F}.get(b0, 0xBF)
    if not lo <= b[i + 1] <= hi:
        return RUNE_ERROR, 1
    for k in range(2, sz):
        if not 0x80 <= b[i + k] <= 0xBF:
            return RUNE_ERROR, 1
    r = b0 & (0x1F, 0x0F, 0x07)[sz - 2]
    for k in range(1, sz):
        r = (r << 6) | (b[i + k] & 0x3F)
    return r, sz


def runes(b):
    out, i = [], 0
    while i < len(b):
        r, sz = decode_rune(b, i)
        out.append(r)
        i += sz
    return out


def _rune_chr(r):
    return chr(r)   # U+FFFD for an invalid byte; surrogates never come out of decode_rune


def regular_match(pat, s):
    """regularMatchForLikeOp(pat, s): replace() turns `\\x` into the literal rune x, a trailing lone `\\` into a literal backslash, `_` into
    `.`, `%` into `.*`, every other rune into itself (regex metacharacters quoted), and matches ^(?s:...)$ against s.  Go's regexp decodes the
    subject with utf8.DecodeRune, so here both sides are decoded the same way and matched as Python strings of those runes."""
    rs = runes(pat)
    out, escaped = [], False
    for r in rs:
        if escaped:
            out.append(re.escape(_rune_chr(r)))
            escaped = False
        elif r == 0x5C:
            escaped = True
        elif r == 0x5F:
            out.append(".")
        elif r == 0x25:
            out.append(".*")
        else:
            out.append(re.escape(_rune_chr(r)))
    if escaped:
        out.append(re.escape("\\"))
    subject = "".join(_rune_chr(r) for r in runes(s))
    return re.fullmatch("(?s:" + "".join(out) + ")", subject) is not None


def remove_escape(src):
    """functionUtil.RemoveEscapeChar(src, '\\\\'): `\\x` -> x; a trailing lone backslash is kept"""
    out, i = bytearray(), 0
    while i < len(src):
        if src[i] == 0x5C and i + 1 < len(src):
            i += 1
        out.append(src[i])
        i += 1
    return bytes(out)


def optimize_rule(pat):
    """optimizeRuleForLike for a non-NULL const pattern: None when it declines, else the byte-level test it applies to every row"""
    n = len(pat)
    if n == 0:
        return lambda v: len(v) == 0                                          # rule 1
    if n == 1:
        if pat == b"%":
            return lambda v: True                                             # 2.1
        if pat == b"_":
            return lambda v: len(v) == 1                                      # 2.2: one byte
        return lambda v: len(v) == 1 and v[0] == pat[0]                       # 2.3
    c0, c1 = pat[0:1], pat[n - 1:n]
    mid = pat[1:n - 1]
    wild = (b"%", b"_")
    if b"_" not in mid and b"%" not in mid:
        if n > 2 and pat[n - 2:n - 1] == b"\\":
            c1 = b"\\"                                                        # the last byte is escaped
        if c0 not in wild and c1 not in wild:                                 # 4.1
            lit = remove_escape(pat)
            return lambda v: v == lit
        if c0 == b"_" and c1 not in wild:                                     # 4.2
            lit = remove_escape(pat[1:])
            return lambda v: len(v) == len(lit) + 1 and v[1:] == lit
        if c0 == b"%" and c1 not in wild:                                     # 4.3
            lit = remove_escape(pat[1:])
            return lambda v: v.endswith(lit)
        if c1 == b"_" and c0 not in wild:                                     # 4.4
            lit = remove_escape(pat[:n - 1])
            return lambda v: len(v) == len(lit) + 1 and v[:len(lit)] == lit
        if c1 == b"%" and c0 not in wild:                                     # 4.5
            lit = remove_escape(pat[:n - 1])
            return lambda v: v.startswith(lit)
        if c0 == b"%" and c1 == b"%":                                         # 4.6
            lit = remove_escape(mid)
            return lambda v: lit in v
        if c0 == b"%" and c1 == b"_":                                         # 4.7
            lit = remove_escape(mid)
            return lambda v: len(v) > 0 and v[:-1].endswith(lit)
        if c0 == b"_" and c1 == b"%":                                         # 4.8
            lit = remove_escape(mid)
            return lambda v: len(v) > 0 and v[1:].startswith(lit)
        return None                                                           # _lit_
    if c0 == b"%" and c1 == b"%" and b"_" not in mid and b"\\%" not in pat:
        subpats = pat[1:].split(b"%")[:-1]                                    # the pieces before every `%`, escapes kept as bytes

        def chain(v):
            for sp in subpats:
                idx = v.find(sp)
                if idx < 0:
                    return False
                v = v[idx + len(sp):]
            return True
        return chain
    return None


def like(s, pat, pat_const=True):
    """likeFn for one row with non-NULL operands"""
    if pat_const:
        f = optimize_rule(pat)
        if f is not None:
            return f(s)
    return regular_match(pat, s)


def compare(op, a, b):
    """op 0 == 1 != 2 > 3 >= 4 < 5 <=, bytes.Equal / bytes.Compare"""
    return (a == b, a != b, a > b, a >= b, a < b, a <= b)[op]


def like_column(values, pats, pat_const, vnulls=None, pnulls=None, skip=None):
    """the whole call: values / pats lists of bytes (pats of length 1 when pat_const), per-row NULL flags, skip = result null bits on entry.
    Returns (results {row: bool} for the evaluated rows, nulls bool list)."""
    n = len(values)
    pat_null = pat_const and pnulls is not None and pnulls[0]
    res, nulls = {}, []
    for i in range(n):
        isnull = bool((skip is not None and skip[i]) or pat_null or (vnulls is not None and vnulls[i])
                      or (not pat_const and pnulls is not None and pnulls[i]))
        nulls.append(isnull)
        if not isnull:
            res[i] = like(values[i], pats[0] if pat_const else pats[i], pat_const)
    return res, nulls
