"""A Python restatement of the reference's conditional values, row by row, with None for NULL:

  caseFn / generalCaseFn / strCaseFn   operatorSet.go:144-316   parameters c1, v1, c2, v2, ...[, else]: the value of the first j whose
                                                                condition is non-NULL and true (NULL when that value is); else ELSE, or NULL
  iffFn                                operatorSet.go:389-      a NULL or false condition takes the else value: CASE with one WHEN and an ELSE
  CoalesceGeneral / CoalesceStr        func_binary.go:938-993   the first non-NULL operand, or NULL
  EvalCase / EvalIff                   evalExpression.go:501-573  the select lists each branch is evaluated under (case_select_lists)

and the byte layout the device writes: a fixed-width NULL row is zero bytes, a string result is what AppendBytes builds (values of up to 23
bytes inline and zero-padded, longer ones into the area in row order), and a skipped row (its result null bit set on entry) keeps its old
bytes.  Operands are lists of length n (a const operand is a list of one element, repeated by `expand`)."""
SKIP = object()   # a row skipped because its result null bit was set on entry


def expand(col, n):
    return list(col) * n if len(col) == 1 else list(col)


def case_fn(conds, values, else_value, n, skip=None):
    """conds / values: lists of operands (bool-or-None / value-or-None); else_value an operand or None (no ELSE)"""
    conds = [expand(c, n) for c in conds]
    values = [expand(v, n) for v in values]
    z = expand(else_value, n) if else_value is not None else None
    out = []
    for i in range(n):
        if skip is not None and skip[i]:
            out.append(SKIP)
            continue
        for c, v in zip(conds, values):
            if c[i] is not None and c[i]:
                out.append(v[i])
                break
        else:
            out.append(z[i] if z is not None else None)
    return out


def iff_fn(cond, a, b, n, skip=None):
    cond, a, b = expand(cond, n), expand(a, n), expand(b, n)
    out = []
    for i in range(n):
        if skip is not None and skip[i]:
            out.append(SKIP)
        else:
            out.append(a[i] if cond[i] is not None and cond[i] else b[i])
    return out


def coalesce(operands, n, skip=None):
    ops = [expand(o, n) for o in operands]
    out = []
    for i in range(n):
        if skip is not None and skip[i]:
            out.append(SKIP)
            continue
        out.append(next((o[i] for o in ops if o[i] is not None), None))
    return out


def case_select_lists(select, conds):
    """EvalCase's select lists: select = the batch's selectList (True = evaluate), conds = the WHEN results as evaluated under them.
    Returns (the list each WHEN is evaluated under, the list each THEN is evaluated under, ELSE's list).  A row takes WHEN j when it is
    still selected and the condition is non-NULL and true."""
    rem = list(select)
    when_lists, then_lists = [], []
    for c in conds:
        when_lists.append(list(rem))
        took = [r and c[i] is not None and bool(c[i]) for i, r in enumerate(rem)]
        then_lists.append(took)
        rem = [r and not t for r, t in zip(rem, took)]
    return when_lists, then_lists, rem


# ---- bytes
def fixed_bytes(out, width, prior):
    """the result bytes: out[i] is bytes of `width`, None (zero bytes) or SKIP (prior's bytes)"""
    b = bytearray()
    for i, v in enumerate(out):
        b += prior[i * width:(i + 1) * width] if v is SKIP else (bytes(width) if v is None else v)
    return bytes(b)


def str_bytes(out, prior_cells):
    """(cells, area) of a string result: AppendBytes over the chosen values; None is the empty inline cell, SKIP keeps prior_cells' cell"""
    cells, area = bytearray(), bytearray()
    for i, v in enumerate(out):
        if v is SKIP:
            cells += prior_cells[24 * i:24 * (i + 1)]
        elif v is None:
            cells += bytes(24)
        elif len(v) <= 23:
            cells += bytes([len(v)]) + v + bytes(23 - len(v))
        else:
            cells += (0xffffffff).to_bytes(4, "little") + len(area).to_bytes(4, "little") + len(v).to_bytes(4, "little") + bytes(12)
            area += v
    return bytes(cells), bytes(area)


def nulls_of(out):
    """the result null flags: NULL and skipped rows"""
    return [v is None or v is SKIP for v in out]
