"""numpy model of a sparse index's posting lists (eps_index_get_sparse_postings), and of how
eps_index_extend_sparse_postings merges the lists of appended rows into them.

postings_model(csr, n) is the layout the header states: the distinct indices of rows [0, n) ascending, their offsets,
and per index the rows that hold it, ascending, with their values.  extend_model restates the device merge
(sparse_inverted.cu: extend_probe_kernel, extend_union_kernel, extend_place_kernel) step by step, so that the CPU tests
can hold it to postings_model on any table."""
import numpy as np


def postings_model(csr, n):
    off, idx, val = csr
    p = int(off[n])
    rows = np.repeat(np.arange(n, dtype=np.int32), np.diff(off[:n + 1]))
    keys = np.asarray(idx[:p], np.int64)
    order = np.argsort(keys, kind="stable")   # rows ascending within a term
    terms, counts = np.unique(keys, return_counts=True)
    ptr = np.zeros(terms.size + 1, np.int64)
    ptr[1:] = np.cumsum(counts)
    return dict(rows=n, terms=terms.astype(np.uint32), ptr=ptr, post_rows=rows[order],
                post_values=np.asarray(val[:p], np.float32)[order])


def extend_model(old, csr, n):
    """The lists `old` (over rows [0, old["rows"])) extended over rows [old["rows"], n), the way the device does it."""
    off, idx, val = csr
    r0 = old["rows"]
    lo, hi = int(off[r0]), int(off[n])
    rows = np.repeat(np.arange(r0, n, dtype=np.int32), np.diff(off[r0:n + 1]))
    keys = np.asarray(idx[lo:hi], np.int64)
    order = np.argsort(keys, kind="stable")
    new_terms, counts = np.unique(keys, return_counts=True)
    new_ptr = np.zeros(new_terms.size + 1, np.int64)
    new_ptr[1:] = np.cumsum(counts)
    new_rows, new_vals = rows[order], np.asarray(val[lo:hi], np.float32)[order]
    if new_rows.size == 0:
        return dict(old, rows=n)
    ot = old["terms"].astype(np.int64)
    # step 1: new terms no old term has; below = their exclusive sum
    o = np.searchsorted(ot, new_terms)
    shared = np.zeros(new_terms.size, bool)
    if ot.size:
        shared = (o < ot.size) & (ot[np.minimum(o, ot.size - 1)] == new_terms)
    below = np.zeros(new_terms.size + 1, np.int64)
    below[1:] = np.cumsum(~shared)
    t = ot.size + int(below[-1])
    # step 2: slots and counts of the union
    terms = np.zeros(t, np.uint32)
    count = np.zeros(t + 1, np.int64)
    j_of_old = np.searchsorted(new_terms, ot)
    old_slot = np.arange(ot.size) + below[j_of_old]
    terms[old_slot] = ot
    count[old_slot] = np.diff(old["ptr"])
    new_slot = o + below[:-1]
    terms[new_slot] = new_terms
    count[new_slot] += np.diff(new_ptr)
    ptr = np.zeros(t + 1, np.int64)
    ptr[1:] = np.cumsum(count[:-1])
    # step 3: old postings open their term's block, new ones close it
    p_all = old["post_rows"].size + new_rows.size
    post_rows = np.zeros(p_all, np.int32)
    post_values = np.zeros(p_all, np.float32)
    for src_rows, src_vals, src_ptr, slot, at_end in ((old["post_rows"], old["post_values"], old["ptr"], old_slot, False),
                                                      (new_rows, new_vals, new_ptr, new_slot, True)):
        p = np.arange(src_rows.size)
        i = np.searchsorted(src_ptr, p, side="right") - 1
        d = ptr[slot[i] + 1] - src_ptr[i + 1] if at_end else ptr[slot[i]] - src_ptr[i]
        post_rows[p + d] = src_rows
        post_values[p + d] = src_vals
    return dict(rows=n, terms=terms, ptr=ptr, post_rows=post_rows, post_values=post_values)


def same_postings(got, want, what):
    """Byte-equal lists: rows covered, terms, offsets, rows and value bits of every posting."""
    assert got["rows"] == want["rows"], "%s: rows covered %d != %d" % (what, got["rows"], want["rows"])
    for key, dt in (("terms", np.uint32), ("ptr", np.int64), ("post_rows", np.int32), ("post_values", np.uint32)):
        a = np.ascontiguousarray(got[key]).view(dt) if key == "post_values" else np.asarray(got[key], dt)
        b = np.ascontiguousarray(want[key]).view(dt) if key == "post_values" else np.asarray(want[key], dt)
        assert a.shape == b.shape and np.array_equal(a, b), "%s: %s differ" % (what, key)
