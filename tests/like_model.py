"""Restatement of the reference's LIKE (engine/query/expr/expr_evaluator.cpp:14-35, :229-241), independent of the
device matcher (like.cu), for the tests.

    like(subject, pattern)        one pair, through Python's re on bytes
    like_many(subjects, patterns) many pairs at once, a DP over bytes vectorised over the pairs

Semantics: an empty pattern matches only the empty subject; the pattern "%" matches every subject; otherwise '%' is
[^\\n\\r]* and '_' is [^\\n\\r] (libstdc++'s ECMAScript '.' excludes both line terminators), every other byte is a
literal, and the match covers the whole subject.  `cross_lines` and `star_special` switch those two rules off; the
tests use the variants to show the golden file tells the readings apart.
"""
import re

import numpy as np

_LINE = (ord("\n"), ord("\r"))


def to_regex(pattern, cross_lines=False):
    any_ = b"." if cross_lines else b"[^\n\r]"
    out = []
    for b in pattern:
        c = bytes([b])
        out.append(any_ + b"*" if c == b"%" else any_ if c == b"_" else re.escape(c))
    return re.compile(b"".join(out), re.DOTALL)


def like(subject, pattern, cross_lines=False, star_special=True):
    if pattern == b"":
        return subject == b""
    if star_special and pattern == b"%":
        return True
    return to_regex(pattern, cross_lines).fullmatch(subject) is not None


def _pad(strings):
    n = max([len(s) for s in strings] + [1])
    m = np.zeros((len(strings), n), np.uint8)
    for i, s in enumerate(strings):
        m[i, :len(s)] = np.frombuffer(s, np.uint8)
    return m, np.array([len(s) for s in strings], np.int64)


def like_many(subjects, patterns, cross_lines=False, star_special=True):
    """like() of every pair (subjects[i], patterns[i]), as a DP over pattern bytes: D[i, k] = the pattern prefix read
    so far matches the first k bytes of subject i."""
    assert len(subjects) == len(patterns)
    N = len(subjects)
    S, ns = _pad(subjects)
    P, npat = _pad(patterns)
    n = S.shape[1]
    term = np.zeros_like(S, bool) if cross_lines else np.isin(S, _LINE)
    term &= np.arange(n)[None, :] < ns[:, None]
    # cnt[i, k] = line terminators among the first k bytes: '%' can move from k' to k >= k' iff cnt is equal
    cnt = np.concatenate([np.zeros((N, 1), np.int64), np.cumsum(term, axis=1)], axis=1)
    D = np.zeros((N, n + 1), bool)
    D[:, 0] = True
    cols = np.arange(n + 1)[None, :]
    rows = np.arange(N)
    for j in range(P.shape[1]):
        live = j < npat
        c = P[:, j]
        star = live & (c == ord("%"))
        lit = live & ~star
        if star.any():
            last = np.maximum.accumulate(np.where(D, cols, -1), axis=1)
            reach = (last >= 0) & (cnt[rows[:, None], np.maximum(last, 0)] == cnt)
            D = np.where(star[:, None], reach, D)
        if lit.any():
            ok = (S == c[:, None]) | ((c == ord("_"))[:, None] & ~term)
            nxt = np.zeros_like(D)
            nxt[:, 1:] = D[:, :-1] & ok
            D = np.where(lit[:, None], nxt, D)
    out = D[rows, ns]
    out[npat == 0] = ns[npat == 0] == 0
    if star_special:
        out |= np.array([p == b"%" for p in patterns], bool)
    return out
