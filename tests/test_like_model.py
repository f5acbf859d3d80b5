"""tests/like_model.py against the reference's own LIKE answers (tests/golden/like.npz, make_like_golden.py)."""
import os

import numpy as np
import pytest

import like_model as lm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "like.npz")


@pytest.fixture(scope="module")
def golden():
    g = np.load(GOLDEN, allow_pickle=False)

    def unpack(off, buf):
        b = buf.tobytes()
        return [b[off[i]:off[i + 1]] for i in range(off.size - 1)]

    return unpack(g["subj_off"], g["subj_bytes"]), unpack(g["pat_off"], g["pat_bytes"]), g["match"].astype(bool)


def _matrix(subj, pats, **kw):
    S = [s for s in subj for _ in pats]
    P = [p for _ in subj for p in pats]
    return lm.like_many(S, P, **kw).reshape(len(subj), len(pats))


def test_golden_covers_the_cases(golden):
    subj, pats, match = golden
    assert len(subj) >= 200 and len(pats) >= 60
    assert b"" in subj and b"" in pats and b"%" in pats and b"%%" in pats
    assert any(b"\n" in p for p in pats) and any(b"\r" in p for p in pats)
    assert any(max(s, default=0) >= 0x80 for s in subj) and max(len(s) for s in subj) >= 300
    assert 0 < match.mean() < 1


def test_regex_model_equals_golden(golden):
    subj, pats, match = golden
    got = np.array([[lm.like(s, p) for p in pats] for s in subj])
    bad = np.argwhere(got != match)
    assert bad.size == 0, [(subj[i], pats[j], bool(match[i, j])) for i, j in bad[:5]]


def test_dp_model_equals_golden(golden):
    subj, pats, match = golden
    got = _matrix(subj, pats)
    bad = np.argwhere(got != match)
    assert bad.size == 0, [(subj[i], pats[j], bool(match[i, j])) for i, j in bad[:5]]


def test_golden_pins_the_line_terminator_rule(golden):
    """'%' and '_' never match '\\n' / '\\r', but the pattern "%" alone matches everything: a model whose wildcards
    cross line terminators, and one without the "%" special case, each disagree with the reference somewhere."""
    subj, pats, match = golden
    crossing = _matrix(subj, pats, cross_lines=True)
    no_special = _matrix(subj, pats, star_special=False)
    assert (crossing != match).any()
    assert (no_special != match).any()
    i, j, k = subj.index(b"a\nb"), pats.index(b"%"), pats.index(b"%%")
    assert match[i, j] and not match[i, k] and crossing[i, k] and not no_special[i, j]
    assert not match[subj.index(b"a\rb"), pats.index(b"a_b")] and match[subj.index(b"a\rb"), pats.index(b"a\rb")]
