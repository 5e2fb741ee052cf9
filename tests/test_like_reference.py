"""The host restatement of LIKE (tests/like_reference.py) against the reference's own known answers (golden/like_kat.json) and against the
quirks of optimizeRuleForLike and regularMatchForLikeOp read off the Go code."""
import json
import os

import pytest

import like_reference as L

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "like_kat.json")))["cases"]


@pytest.mark.parametrize("case", KAT, ids=lambda c: c["source"].rsplit("/", 1)[-1] + ":" + c["pat"])
def test_known_answers(case):
    s, p = bytes.fromhex(case["str"]), bytes.fromhex(case["pat"])
    got = L.regular_match(p, s) if case["tier"] == "regular" else L.like(s, p, pat_const=True)
    assert (not got if case["not"] else got) == case["expected"]


def test_known_answers_cover_both_tiers():
    like_rows = [bytes.fromhex(c["pat"]) for c in KAT if c["tier"] == "like"]
    assert sum(L.optimize_rule(p) is not None for p in like_rows) >= 20
    assert sum(L.optimize_rule(p) is None for p in like_rows) >= 5
    assert any(c["tier"] == "regular" for c in KAT)


# (subject, pattern, const-pattern result, column-pattern result)
QUIRKS = [
    # `\%`: n == 2, so the escape rule does not fire; rule 4.5 with RemoveEscapeChar("\\") = "\\" (a trailing lone backslash is kept)
    (b"\\abc", b"\\%", True, False),
    (b"%", b"\\%", False, True),
    # `a\_`: the next-to-last byte is a backslash, so the last byte is a literal: rule 4.1 with the literal "a_"
    (b"a_", b"a\\_", True, True),
    (b"ab", b"a\\_", False, False),
    # a trailing lone backslash is a literal in both tiers
    (b"ab\\", b"ab\\", True, True),
    (b"ab", b"ab\\", False, False),
    # tier A's `_` is one byte, tier B's one rune
    ("é".encode(), b"_", False, True),
    ("xé".encode(), b"x_", False, True),
    ("éx".encode(), b"_x", False, True),
    ("xé".encode(), b"%\xc3_", True, False),
    # _lit_ has no rule: rune level even for a const pattern
    ("éabcé".encode(), b"_abc_", True, True),
    (b"xabcy", b"_abc_", True, True),
    # the multi-% chain keeps escapes as bytes; the rune matcher removes them
    (b"xa\\bxc", b"%a\\b%c%", True, False),
    (b"xabxc", b"%a\\b%c%", False, True),
    (b"cxa", b"%a%c%", False, False),
    (b"axc", b"%a%c%", True, True),
    (b"aa", b"%a%%a%", True, True),
    # `\%` in a chain-shaped pattern declines the chain: rune level
    (b"x%yz", b"%\\%%z%", True, True),
    (b"xyz", b"%\\%%z%", False, False),
    # `_` in the middle declines the chain
    ("aéb".encode(), b"%a_b%", True, True),
    # rule 4.7 / 4.8 edge: the wildcard byte must exist
    (b"", b"%_", False, False),
    (b"a", b"_%", True, True),
    (b"", b"", True, True),
    (b"a", b"", False, False),
    # an invalid pattern byte is U+FFFD, which matches U+FFFD and any invalid subject byte (rune level; tier A compares bytes)
    (b"a\xfex", b"a\xff_", False, True),
    ("a�x".encode(), b"a\xff_", False, True),
    (b"a\xffx", b"a\xff_", True, True),
    # overlong and surrogate sequences are one RuneError per byte
    (b"\xed\xa0\x80", b"___", True, True),
    (b"\xc0\xaf", b"__", True, True),
    (b"\xc0\xaf", b"_", False, False),
    # embedded zero bytes and newlines are ordinary bytes / runes; `%` crosses newlines
    (b"a\x00b", b"a_b", True, True),
    (b"a\nb\nc", b"a%c", True, True),
    # regex metacharacters are literals
    (b"a.b", b"a.b", True, True),
    (b"axb", b"a.b", False, False),
]


@pytest.mark.parametrize("s,p,const_res,col_res", QUIRKS)
def test_quirks(s, p, const_res, col_res):
    assert L.like(s, p, pat_const=True) == const_res
    assert L.like(s, p, pat_const=False) == col_res


def test_decode_rune_matches_python_on_valid_utf8():
    for text in ["", "abc", "é", "中文", "\U0001F600x", "�"]:
        assert L.runes(text.encode()) == [ord(c) for c in text]


def test_compare_is_bytes_order():
    assert L.compare(4, b"ab", b"abc") and L.compare(2, b"\xff", b"\x00\x01")
    assert L.compare(0, b"a\x00", b"a\x00") and L.compare(1, b"a", b"a\x00")
    assert L.compare(5, b"", b"")
