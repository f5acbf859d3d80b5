"""Exact CPU model of the dense graph search at any search width W, and tables whose distances are exact in any order.

Integer tables.  Rows and queries hold small integers, |v| <= B.  Every partial sum of an L2 distance, of the expanded
form |x|^2 - 2 x.q + |q|^2 a tile kernel may use, and of an inner product is an integer of magnitude at most
d (2B)^2.  While that is below 2^24 every fp32 partial sum is exact, so every kernel, whatever its summation order and
with or without FMA, returns the same integer distance; cosine (1 - x.q over the stored rows; the index does not
normalise) and IP (-x.q) hold for the same reason.  B = 8 allows d < 65 536.  `assert_exact` checks the bound for a
table and its queries.  Integer distances tie often, which exercises the (distance, id) order everywhere.

Search at width W (graph_search.cu, DESIGN.md §K2).  Seed the queue with prepare_init_ids and sort it by (distance, id).
Each step takes the first min(W, #unchecked) unchecked queue entries and marks them checked, tests-and-sets every id of
their full CSR rows against one visited set, computes the distances of the fresh ids, and keeps the best L of the
queue and the fresh ids by (distance, id), checked flags kept.  The search stops when nothing is unchecked.  At W = 1
this is SearchImpl at IntraQueryThreads = 1 (the oracle port).  `search` adds the Search wrapper: L clamp, tail scan
merged with merge_fixed, post-filter on deleted rows and the filter, L_local and limit, and the brute branch below 512
indexed rows."""
import numpy as np

EXACT_SUM_LIMIT = 1 << 24  # fp32 represents every integer of magnitude <= 2^24
BRUTE_BELOW = 512          # BruteforceThreshold: fewer indexed rows take the exact scan
METRICS = ("l2", "ip", "cosine")


def int_table(n, d, seed, B=8):
    """n x d float32 rows of uniform integers in [-B, B]."""
    rng = np.random.default_rng(seed)
    return rng.integers(-B, B + 1, size=(n, d)).astype(np.float32)


def assert_exact(X, Q):
    """Every fp32 distance between rows of X and Q is an exact integer under any summation order."""
    d = X.shape[1]
    B = max(float(np.abs(X).max(initial=0)), float(np.abs(Q).max(initial=0)))
    assert np.all(X == np.round(X)) and np.all(Q == np.round(Q)), "table holds non-integers"
    assert d * (2 * B) ** 2 < EXACT_SUM_LIMIT, "d (2B)^2 = %g reaches 2^24" % (d * (2 * B) ** 2)


def distances(metric, X, ids, q):
    """fp32 distances of rows X[ids] to q.  float64 arithmetic is exact on integer tables (assert_exact)."""
    R = X[ids].astype(np.float64)
    q = q.astype(np.float64)
    if metric == "l2":
        v = ((R - q) ** 2).sum(1)
    elif metric == "ip":
        v = -(R @ q)
    else:
        v = 1.0 - R @ q
    return (v.astype(np.float32) + np.float32(0)).astype(np.float32)  # -0 folds into +0, as every comparison does


def keys_of(dist, ids):
    """uint64 keys ordered as (distance, id): the device's [ordered float : 32][0 : 1][id : 31]."""
    u = (np.asarray(dist, np.float32) + np.float32(0)).view(np.uint32).astype(np.uint64)
    o = np.where(u & np.uint64(0x80000000), ~u & np.uint64(0xffffffff), u | np.uint64(0x80000000))
    return (o << np.uint64(32)) | np.asarray(ids, np.uint64)


def key_ids(k):
    return (k & np.uint64(0x7fffffff)).astype(np.int64)


def key_dists(k):
    o = (k >> np.uint64(32)).astype(np.uint32)
    u = np.where(o & np.uint32(0x80000000), o & np.uint32(0x7fffffff), ~o)
    return u.astype(np.uint32).view(np.float32)


def prepare_init_ids(off, nb, nav, n_indexed, L):
    """PrepareInitIds: the distinct out-neighbours of the navigation point, then nav + 1, nav + 2, ... (mod n)."""
    row = nb[off[nav]:off[nav + 1]]
    _, first = np.unique(row, return_index=True)
    head = row[np.sort(first)][:L]
    sel = np.zeros(n_indexed, bool)
    sel[head] = True
    ring = (nav + 1 + np.arange(n_indexed)) % n_indexed
    rest = ring[~sel[ring]][:L - head.size]
    return np.concatenate([head, rest]).astype(np.int64)


class QueryRun:
    """What one query's search produced: the final queue (keys, checked flags), its counters and the number of fresh
    ids it found (what the device logs and tests against its visited-set limits)."""
    __slots__ = ("keys", "checked", "n_dist", "n_expand", "n_edges", "fresh")


def wide_search(X, q, metric, graph, L, W, init_ids=None, corrupt=None):
    """Search one query at width W over graph = (n_indexed, offsets, nbrs, nav) with queue length L <= n_indexed.

    `corrupt` seeds one deliberate fault, to show that the comparisons catch it: "tie" compares a fresh row with the
    worst queue entry by distance alone (a row tying it with a smaller id is rejected), "skip" drops the first fresh id
    of every step, "second" picks the second unchecked entry when there are two.  (Accepting on key <= bound instead
    of key < bound is no fault: a fresh id is never in the queue, so no key equals the bound.)"""
    n_indexed, off, nb, nav = graph
    if init_ids is None:
        init_ids = prepare_init_ids(off, nb, nav, n_indexed, L)
    visited = np.zeros(n_indexed, bool)
    visited[init_ids] = True
    keys = np.sort(keys_of(distances(metric, X, init_ids, q), init_ids))
    checked = np.zeros(L, bool)
    r = QueryRun()
    r.n_dist, r.n_expand, r.n_edges, r.fresh = L, 0, 0, 0
    cursor = 0  # every entry before it is checked
    while True:
        unc = np.flatnonzero(~checked[cursor:]) + cursor
        if unc.size == 0:
            break
        cursor = int(unc[0])
        pick = unc[:W]
        if corrupt == "second" and unc.size > 1:
            pick = unc[1:W + 1]
        checked[pick] = True
        r.n_expand += pick.size
        cids = key_ids(keys[pick])
        rows = [nb[off[c]:off[c + 1]] for c in cids]
        ids = np.concatenate(rows) if rows else np.zeros(0, np.int64)
        r.n_edges += ids.size
        u, first = np.unique(ids, return_index=True)
        fresh = u[~visited[u]]
        visited[fresh] = True
        if corrupt == "skip" and fresh.size:
            fresh = np.setdiff1d(fresh, ids[np.sort(first[np.isin(u, fresh)])][:1])
        r.n_dist += fresh.size
        r.fresh += fresh.size
        if fresh.size == 0:
            continue
        fk = np.sort(keys_of(distances(metric, X, fresh, q), fresh))
        if corrupt == "tie":
            fk = fk[(fk >> np.uint64(32)) < (keys[L - 1] >> np.uint64(32))]
        fk = fk[fk < keys[L - 1]]
        if fk.size == 0:
            continue
        at = np.searchsorted(keys, fk)
        keys = np.insert(keys, at, fk)[:L]
        checked = np.insert(checked, at, False)[:L]
        cursor = min(cursor, int(at[0]))
    r.keys, r.checked = keys, checked
    return r


def merge_fixed(keys, n1, tail_keys):
    """MergeTwoQueuesInto1stQueueSeqFixed: the first n1 entries become the best n1 of themselves and the (sorted,
    id-disjoint) tail keys; entries from n1 on are left as they were."""
    if tail_keys.size == 0 or n1 == 0:
        return keys
    head = np.sort(np.concatenate([keys[:n1], tail_keys]))[:n1]
    return np.concatenate([head, keys[n1:]])


class Result:
    __slots__ = ("ids", "dists", "counts", "n_dist", "n_expand", "n_edges", "n_seed", "runs")


def search(X, Q, metric, graph, L_master, limit, W=1, L_local=None, total=None, deleted=None, keep=None, corrupt=None):
    """Search of every query of Q.  X holds all `total` rows; graph covers [0, n_indexed).  `deleted` is a bool mask
    over rows, `keep(ids, dists)` the filter.  L_local defaults to L_master, and the merge window is clamped to the
    queue length.  Returns ids [nq x limit] (-1 padded), dists float64 (inf padded), counts, and per query n_dist,
    n_expand, n_edges, n_seed, plus the QueryRun of each graph search."""
    n_indexed, off, nb, nav = graph
    total = X.shape[0] if total is None else total
    L_local = L_master if L_local is None else L_local
    nq = Q.shape[0]
    out = Result()
    out.ids = np.full((nq, limit), -1, np.int64)
    out.dists = np.full((nq, limit), np.inf, np.float64)
    out.counts = np.zeros(nq, np.int64)
    for f in ("n_dist", "n_expand", "n_edges", "n_seed"):
        setattr(out, f, np.zeros(nq, np.int64))
    out.runs = []

    def admissible(ids, ds):
        ok = np.ones(ids.size, bool)
        if deleted is not None:
            ok &= ~deleted[ids]
        if keep is not None:
            ok &= keep(ids, ds)
        return ok

    def scan(q, start, end):
        ids = np.arange(start, end, dtype=np.int64)
        ds = distances(metric, X, ids, q)
        ok = admissible(ids, ds)
        return np.sort(keys_of(ds[ok], ids[ok]))

    brute = n_indexed < BRUTE_BELOW
    L = min(L_master, n_indexed)
    search_limit = min(n_indexed, limit, L_local, L)
    init_ids = None if brute else prepare_init_ids(off, nb, nav, n_indexed, L)
    for qi in range(nq):
        q = Q[qi]
        if brute:
            k = scan(q, 0, total)[:min(limit, L_local)]
            out.n_dist[qi] = total
        else:
            run = wide_search(X, q, metric, graph, L, W, init_ids=init_ids, corrupt=corrupt)
            out.runs.append(run)
            out.n_dist[qi], out.n_expand[qi], out.n_edges[qi], out.n_seed[qi] = run.n_dist, run.n_expand, run.n_edges, L
            keys = run.keys
            if total > n_indexed:
                tk = scan(q, n_indexed, total)[:limit]
                out.n_dist[qi] += total - n_indexed
                keys = merge_fixed(keys, search_limit, tk)
            ids, ds = key_ids(keys), key_dists(keys)
            k = keys[admissible(ids, ds)][:search_limit]
        out.counts[qi] = k.size
        out.ids[qi, :k.size] = key_ids(k)
        out.dists[qi, :k.size] = key_dists(k)
    return out


def random_csr(n, deg_lo, deg_hi, seed, self_loops=0.0, dup=0.0):
    """CSR with row degrees uniform in [deg_lo, deg_hi]; a share `self_loops` of the rows list themselves and a share
    `dup` of the ids repeat an earlier id of their row."""
    rng = np.random.default_rng(seed)
    deg = rng.integers(deg_lo, deg_hi + 1, n)
    off = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    nb = rng.integers(0, n, off[-1]).astype(np.int64)
    for v in np.flatnonzero(rng.random(n) < self_loops):
        if deg[v]:
            nb[off[v] + rng.integers(deg[v])] = v
    for e in np.flatnonzero(rng.random(off[-1]) < dup):
        v = np.searchsorted(off, e, side="right") - 1
        if e > off[v]:
            nb[e] = nb[rng.integers(off[v], e)]
    return off, nb


def with_rows(off, nb, rows):
    """The CSR with the rows of the vertices in `rows` ({vertex: ids}) replaced."""
    n = off.size - 1
    parts = [nb[off[v]:off[v + 1]] if v not in rows else np.asarray(rows[v], np.int64) for v in range(n)]
    deg = np.array([p.size for p in parts], np.int64)
    return np.concatenate([[0], np.cumsum(deg)]).astype(np.int64), np.concatenate(parts).astype(np.int64)


# The device's visited hash set (graph_search.cu prepare_visited, graph_search.cuh vset_bucket)
VSET_MUL = 0x9e3779b1


def vset_geometry(L):
    """(entries, bucket shift, entries a query may insert before it moves to the bitmap) of the table for queue L."""
    cap = min(16384, max(1024, 1 << (16 * L - 1).bit_length()))
    return cap, 32 - (cap.bit_length() - 1 - 3), cap // 4 * 3


def vset_bucket(ids, L):
    """First entry of each id's 8-entry bucket."""
    _, shift, _ = vset_geometry(L)
    h = (np.asarray(ids, np.uint64) * np.uint64(VSET_MUL)) & np.uint64(0xffffffff)
    return ((h >> np.uint64(shift)) << np.uint64(3)).astype(np.int64)
