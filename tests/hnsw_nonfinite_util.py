"""Non-finite HNSW test cases (test infrastructure), shared by the CPU and GPU tests and tests/golden/make_golden_hnsw_nonfinite.py.

An index is built from FINITE rows (so no builder ever sees a NaN); then the stored feature values of chosen nodes are
overwritten in the saved index.mmap_store.  The graph stays the finite one and only distances change.  Rows and queries are
chosen so that each non-finite class is forced whatever the summation order: products that overflow on their own (1e20 x
+-1e20), a NaN component, inf x an explicitly stored 0.0.  One row overflows only in the reference's avx512 lane order: two
+1.8e38 products in SIMD lane j (components j, j + 16) and two -1.8e38 products in lane k (k, k + 16): lane sums +inf and -inf,
folded to NaN, where a left-to-right sum stays finite.  Opposite overflows only force NaN where both products are rounded on
their own: in the fused scalar tail fma(1e20, -1e20, +inf) = +inf, so the rows that overflow both ways keep their two
overflowing products out of the tail.

Dense rows: every special component is zero in the finite rows; the overwritten components sit in the 64-wide main chunks, the
4-wide remainder and the fused scalar tail (SPOTS).  Sparse rows: values are overwritten at stored entries only.
"""
import numpy as np
import scipy.sparse as smat

BIG = np.float32(1e20)      # |BIG x BIG| > FLT_MAX: overflows in float32 on its own
HALF_LANE = np.float32(1.8e18)  # BIG x HALF_LANE = 1.8e38: two of them overflow, one does not
FLT_MAX = float(np.finfo(np.float32).max)
EPS32 = 2.0 ** -24
ORDER_J, ORDER_K = 1, 2     # SIMD lanes of the order-dependent row (components j, j + 16 and k, k + 16)


# ------------------------------------------------------------------------------------------------ the saved index file
def _l0_block(path):
    """(raw bytes of index.mmap_store, byte offset of the level-0 buffer in the file) (mmap_util.hpp layout, block 13)."""
    raw = np.fromfile(path, dtype=np.uint8)
    meta_off = int(raw[-8:].view(np.uint64)[0])
    info = raw[meta_off + 8: meta_off + 8 + 16 * 14].view(np.uint64).reshape(14, 2)
    return raw, int(info[13, 0])


def overwrite_values(folder, edits):
    """edits: {node: {component (dense) or stored column index (sparse): value}} -> written into <folder>/c_model/index.mmap_store."""
    import os

    from oracle.restatement import OracleHNSW

    o = OracleHNSW(folder)
    path = os.path.join(folder, "c_model", "index.mmap_store")
    raw, off = _l0_block(path)
    head = (1 + o.l0_max_degree) * 4
    for node, vals in edits.items():
        if o.sparse:
            b = off + int(o.mem_start[node]) + head
            n = int(raw[b:b + 4].view(np.uint32)[0])
            cols = raw[b + 4 + 4 * n:b + 4 + 8 * n].view(np.uint32)
            for c, v in vals.items():
                at = np.flatnonzero(cols == c)
                assert at.size == 1, f"node {node} does not store column {c}"
                raw[b + 4 + 4 * int(at[0]):b + 8 + 4 * int(at[0])] = np.array([v], np.float32).view(np.uint8)
        else:
            b = off + node * o.l0_node_mem + head + 4
            for c, v in vals.items():
                raw[b + 4 * c:b + 4 * c + 4] = np.array([v], np.float32).view(np.uint8)
    raw.tofile(path)


def top_level_nodes(o):
    """Nodes on the top level of the restatement's parsed index: the entry node and every neighbour listed there."""
    nodes = {o.init_node}
    if o.max_level == 0:
        return sorted(nodes)
    l1 = o.l1.view(np.uint32)
    for r in range(o.num_node):
        b = r * (o.l1_node_mem // 4) + (o.max_level - 1) * (o.l1_level_mem // 4)
        deg = min(int(l1[b]), o.l1_max_degree)
        nodes |= set(int(x) for x in l1[b + 1:b + 1 + deg])
    return sorted(nodes)


# ------------------------------------------------------------------------------------------------------- dense cases
def spots(d):
    """Components in each part of a row of width d: the main chunks (first and last 16-block), the 4-wide remainder and the
    scalar tail (where d has them), never an order-dependent component."""
    m = 16 * (d // 16)
    tl = d - m
    out = [0, 3] if m else []
    if m >= 32:
        out += [m - 1, m - 5]
    if tl >= 4:
        out += [m, m + 3]
    if tl % 4:
        out += [d - 1]
    order = {ORDER_J, ORDER_J + 16, ORDER_K, ORDER_K + 16}
    return [c for c in out if c not in order]


def dense_rows(rng, n, d):
    """Finite unit rows with every special component 0."""
    X = rng.standard_normal((n, d)).astype(np.float32)
    X[:, special_components(d)] = 0
    return (X / np.linalg.norm(X, axis=1, keepdims=True)).astype(np.float32)


def special_components(d):
    s = set(spots(d))
    if d >= 32:
        s |= {ORDER_J, ORDER_J + 16, ORDER_K, ORDER_K + 16}
    return sorted(s)


def inf_component(d):
    """A component that is NOT special (the finite rows hold non-zero values there) for the query with an inf component."""
    return next(c for c in range(d) if c not in set(special_components(d)))


def dense_edits(o, d, metric, variant):
    """Overwrites of one dense index (parsed by the restatement, o): {node: {component: value}}, and the kind of each node.
    variant "scattered": NaN rows on the top level and NaN / +inf / -inf / both / inf x 0 rows over level 0;
    "entry_nan": a NaN at the entry node; "entry_neginf": a -inf ip distance at the entry node for the overflow query."""
    sp = spots(d)
    ci = inf_component(d)
    # both overflows of a NaN row sit on components that are multiplied un-fused: in the fused scalar tail the product is not
    # rounded on its own, so fma(1e20, -1e20, +inf) = +inf and such a row would be +-inf, not NaN
    m, tl = 16 * (d // 16), d % 16
    unfused = [c for c in sp if c < m + 4 * (tl // 4)]
    edits, kinds = {}, {}
    if variant == "entry_nan":
        edits[o.init_node] = {sp[-1]: np.float32(np.nan)}
        kinds[o.init_node] = "nan"
        return edits, kinds
    if variant == "entry_neginf":
        edits[o.init_node] = {c: BIG for c in sp}
        kinds[o.init_node] = "pos"
        return edits, kinds
    top = [n for n in top_level_nodes(o) if n != o.init_node][:3]
    rest = [n for n in range(o.num_node) if n != o.init_node and n not in top]
    rng = np.random.default_rng(d * 7 + (metric == "l2"))
    pick = list(rng.choice(rest, size=min(len(rest), 48), replace=False))
    for i, n in enumerate(top):
        edits[int(n)] = {sp[i % len(sp)]: np.float32(np.nan)}
        kinds[int(n)] = "nan"
    for i, n in enumerate(pick):
        c = sp[i % len(sp)]
        kind = ("nan", "pos", "neg", "both", "zero", "pos", "neg", "order")[i % 8]
        if kind == "nan":
            e = {c: np.float32(np.nan)}
        elif kind == "pos":
            e = {c: BIG}
        elif kind == "neg":
            e = {c: -BIG}
        elif kind == "both":
            e = {unfused[0]: BIG, unfused[-1]: -BIG}
        elif kind == "zero":  # an explicit 0.0 where the query with an inf component has it: inf x 0 = NaN
            e = {ci: np.float32(0.0)}
        else:
            if d < 32:
                e = {c: BIG}
            else:
                e = {ORDER_J: HALF_LANE, ORDER_J + 16: HALF_LANE, ORDER_K: -HALF_LANE, ORDER_K + 16: -HALF_LANE}
        edits[int(n)] = e
        kinds[int(n)] = kind
    return edits, kinds


def dense_queries(rng, d, nq=12):
    """Finite queries (every special component 0), then: the overflow query (BIG on the spots), a query with a NaN component,
    one with an inf component, and (d >= 32) the query that meets the order-dependent row (BIG on its four components).
    Returns (Q, index of the order query or None)."""
    Q = rng.standard_normal((nq + 4, d)).astype(np.float32)
    Q[:, special_components(d)] = 0
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    Q[nq, spots(d)] = BIG
    Q[nq + 1, d // 2] = np.nan
    Q[nq + 2, inf_component(d)] = np.inf
    order_q = None
    if d >= 32:
        Q[nq + 3, [ORDER_J, ORDER_J + 16, ORDER_K, ORDER_K + 16]] = BIG
        order_q = nq + 3
    return np.ascontiguousarray(Q, dtype=np.float32), order_q


def apply_dense(X, edits):
    X = X.copy()
    for n, e in edits.items():
        for c, v in e.items():
            X[n, c] = v
    return X


# ------------------------------------------------------------------------------------------------------ sparse cases
SP_D = 6000                       # > 4,096: one query row is searched from global memory
SP_COLS = (0, 1, 2, 3, 4)         # 0, 1: overflow; 2: inf x stored 0.0; 3: NaN on a matched index; 4: NaN on an unmatched one


def sparse_rows(rng, n, nnz=12):
    """Finite csr rows over SP_D columns (column indices >= 5, values in (0.1, 1.1)); every 4th row also stores columns 0..4
    (value 0.5), the entries the edits overwrite."""
    indptr, idx, val = [0], [], []
    for i in range(n):
        c = np.sort(rng.choice(np.arange(5, SP_D), size=nnz, replace=False))
        if i % 4 == 0:
            c = np.concatenate([np.array(SP_COLS), c])
        idx.append(c)
        val.append(np.where(c < 5, 0.5, rng.random(c.size) + 0.1).astype(np.float32))
        indptr.append(indptr[-1] + c.size)
    return smat.csr_matrix((np.concatenate(val), np.concatenate(idx), indptr), shape=(n, SP_D), dtype=np.float32)


def sparse_edits(X, seed):
    """NaN on a matched index (3) and on an unmatched one (4), overflowing products (0: BIG, 1: -BIG, both), a stored 0.0
    under the query's inf (2), on rows that store columns 0..4."""
    rng = np.random.default_rng(seed)
    holders = [r for r in range(X.shape[0]) if X.indptr[r + 1] - X.indptr[r] > 12]
    pick = list(rng.choice(holders, size=min(len(holders), 40), replace=False))
    edits = {}
    for i, n in enumerate(pick):
        kind = i % 6
        edits[int(n)] = [{3: np.float32(np.nan)}, {4: np.float32(np.nan)}, {0: BIG}, {1: -BIG}, {0: BIG, 1: -BIG},
                         {2: np.float32(0.0)}][kind]
    return edits


def sparse_queries(rng, nq=12):
    """Finite queries (columns >= 5, a few also column 3 or 4 with finite values); the overflow query (BIG on columns 0, 1);
    one with inf on column 2; one with a NaN on a column >= 5; and one of 5,000 entries (global-memory search) carrying a
    NaN and column 3."""
    rows = []
    for i in range(nq):
        c = np.sort(rng.choice(np.arange(5, SP_D), size=40, replace=False))
        if i % 3 == 0:
            c = np.concatenate([[3], c])
        rows.append((c, (rng.random(c.size) + 0.1).astype(np.float32)))
    c = np.sort(rng.choice(np.arange(5, SP_D), size=40, replace=False))
    rows.append((np.concatenate([[0, 1], c]), np.concatenate([[BIG, BIG], rng.random(c.size) + 0.1]).astype(np.float32)))
    rows.append((np.concatenate([[2], c]), np.concatenate([[np.inf], rng.random(c.size) + 0.1]).astype(np.float32)))
    v = (rng.random(c.size) + 0.1).astype(np.float32)
    v[c.size // 2] = np.nan
    rows.append((c, v))
    c = np.concatenate([[3], np.sort(rng.choice(np.arange(5, SP_D), size=4999, replace=False))])
    v = (rng.random(c.size) + 0.1).astype(np.float32)
    v[100] = np.nan
    rows.append((c, v))
    indptr = np.cumsum([0] + [r[0].size for r in rows])
    Q = smat.csr_matrix((np.concatenate([r[1] for r in rows]), np.concatenate([r[0] for r in rows]), indptr),
                        shape=(len(rows), SP_D), dtype=np.float32)
    return Q


def apply_sparse(X, edits):
    X = X.copy()
    for n, e in edits.items():
        for c, v in e.items():
            at = X.indptr[n] + int(np.flatnonzero(X.indices[X.indptr[n]:X.indptr[n + 1]] == c)[0])
            X.data[at] = v
    return X


# -------------------------------------------------------------------------------------------------------------- checks
def assert_same_nan_hnsw(got, want, what=""):
    """ids bit-equal; distances bit-equal except that two NaNs (of any payload) are equal."""
    from .util import assert_same_nan

    assert_same_nan(got, want, what, tags="ID")


def f64_check(X, Q, metric, idx, dist, skip=(), what=""):
    """Every returned (query, id) against a float64 evaluation: finite distances within 2 m 2^-24 sum|term| + one ulp of the
    float32 result; the classes that overflowing or NaN terms force exactly (NaN, +inf, -inf).  Sparse "l2" is the reference's
    (|x - x|^2 + |y - y|^2) - 2<x,y>: NaN as soon as either row stores a NaN or +-inf, matched or not.  `skip`: (query, node) pairs
    whose class depends on the summation order."""
    sparse = smat.issparse(X)
    skip = set(skip)
    n_checked = 0
    for q in range(Q.shape[0]):
        rows = idx[q].astype(np.int64)
        g = dist[q].astype(np.float64)
        valid = ~((idx[q] == 0) & (dist[q].view(np.uint32) == 0))
        if sparse:
            qv = np.zeros(X.shape[1])
            has = np.zeros(X.shape[1], bool)
            Qr = Q[q]
            qv[Qr.indices] = Qr.data
            has[Qr.indices] = True
            terms = []
            for r in rows:
                s = X[int(r)]
                h = has[s.indices]
                terms.append(s.data[h].astype(np.float64) * qv[s.indices[h]])
        else:
            xq = np.asarray(Q[q], np.float64)
            terms = [(X[int(r)].astype(np.float64) - xq) ** 2 if metric == "l2" else X[int(r)].astype(np.float64) * xq
                     for r in rows]
        with np.errstate(invalid="ignore", over="ignore"):
            for j, (r, t) in enumerate(zip(rows, terms)):
                if not valid[j] or (q, int(r)) in skip:
                    continue
                nan = np.isnan(t).any() or ((t > FLT_MAX).any() and (t < -FLT_MAX).any())
                if sparse and metric == "l2":  # the reference adds the squared norms |x - x|^2 + |y - y|^2: NaN for a non-finite entry
                    nan = nan or not np.isfinite(X[int(r)].data).all() or not np.isfinite(Q[q].data).all()
                pos, neg = (t > FLT_MAX).any(), (t < -FLT_MAX).any()
                s = float(t.sum()) if t.size else 0.0
                l2_dense = metric == "l2" and not sparse
                scale = 1.0 if l2_dense else (1.0 if metric == "ip" else 2.0)
                d64 = s if l2_dense else (1.0 - s if metric == "ip" else -2.0 * s)
                if nan:
                    assert np.isnan(g[j]), f"{what} q={q} node={r}: want NaN, got {g[j]}"
                elif pos or neg:
                    want = np.inf if (l2_dense or neg) else -np.inf
                    assert g[j] == want, f"{what} q={q} node={r}: want {want}, got {g[j]}"
                else:
                    bnd = 2 * max(t.size, 1) * EPS32 * scale * float(np.abs(t).sum()) + float(np.spacing(np.float32(abs(d64))))
                    assert abs(g[j] - d64) <= bnd, f"{what} q={q} node={r}: {g[j]} vs float64 {d64} (bound {bnd})"
                n_checked += 1
    return n_checked
