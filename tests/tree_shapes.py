"""TEST INFRASTRUCTURE: spanning trees whose SHAPE reaches the limits of the tree filter's BFS and level walk
(``csrc/tree_filter.cu``), the canonical BFS order of any root, and a float64 restatement of the refine recursion.

Every builder is seeded numpy and returns ``(edges, (h, w))``: int32 ``[V-1, 2]`` edges of a spanning tree of the
``h x w`` map (V = h * w, vertex ``r * w + c``).  Levels are counted from vertex 0 unless stated otherwise.

- ``path(n)``: the 1 x n row; n levels from vertex 0, two vertices per level from the centre.
- ``serpentine(h, w)``: the rows joined at alternating ends; a Hamiltonian path, so L = V from a corner.
- ``comb(h, w)``: spine = column 0, teeth = the rows.  Level k from (0, 0) is the anti-diagonal r + c = k: every width
  from 1 to min(h, w) occurs and L = h + w - 1.
- ``htree(m, widest)``: the H-tree fractal on the (2^(m+1) - 1)^2 grid (its 4^m tips all at depth 2^(m+1) - 2 from
  the centre), the other cells attached by a breadth-first flood from the H.  A 4-connected grid tree.
- ``broom(path_len, widths)``: a path, then levels of the given widths (at most 3 children per vertex, 4 for the
  root); vertex ids shuffled, so no grid structure.  Reaches (L, width) pairs no grid tree of that size can.
- ``random_mst(h, w)``: the MST of random grid weights, as a control.

The limits below restate the launch rules of ``csrc/tree_filter.cu`` from its constants."""
import numpy as np

# ---- limits, restated from csrc/tree_filter.cu ----
BFS_FRONT = 1024                          # frontier entries of bfs_grid_kernel; a wider level declines to bfs_block_kernel
_BFS_BUFS, _BFS_STRIDE = 4, BFS_FRONT + 32
_MAX_TREE_SMEM = 220 * 1024
PF, RW, RNT, LWIN, LCHUNK = 6, 128, 256, 1024, 256
_RING_BYTES = PF * RW * (16 + 4 + 4) + LWIN * 4        # sizeof(RingSmem): float4 q, int ia, float fa per slot + window
_MAX_REFINE_SMEM = 227 * 1024 - _RING_BYTES - 64


def grid_bfs_tried(V):
    """bxs_bfs_forward_rooted launches bfs_grid_kernel iff its shared memory (V adjacency bytes rounded up to words,
    plus the frontier buffers) fits."""
    return ((V + 3) // 4) * 4 + _BFS_BUFS * 2 * _BFS_STRIDE * 4 <= _MAX_TREE_SMEM


def refine_in_smem(V):
    """The refine kernels keep the position-ordered values in shared memory iff V + 4 floats fit beside the ring."""
    return (V + 4) * 4 <= _MAX_REFINE_SMEM


GRID_BFS_MAX_V = max(v for v in range(190000, 193000) if grid_bfs_tried(v))
REFINE_SMEM_MAX_V = max(v for v in range(52000, 53000) if refine_in_smem(v))


# ---- builders ----
def _e(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.int64).reshape(-1, 2).astype(np.int32))


def path(n):
    v = np.arange(n - 1)
    return _e(np.stack([v, v + 1], 1)), (1, n)


def serpentine(h, w):
    ids = np.arange(h * w).reshape(h, w)
    hori = np.stack([ids[:, :-1], ids[:, 1:]], -1).reshape(-1, 2)
    cols = np.where(np.arange(h - 1) % 2 == 0, w - 1, 0)            # row r joins row r + 1 at its far end
    vert = np.stack([ids[:-1][np.arange(h - 1), cols], ids[1:][np.arange(h - 1), cols]], 1)
    return _e(np.concatenate([hori, vert])), (h, w)


def comb(h, w):
    ids = np.arange(h * w).reshape(h, w)
    hori = np.stack([ids[:, :-1], ids[:, 1:]], -1).reshape(-1, 2)
    spine = np.stack([ids[:-1, 0], ids[1:, 0]], 1)
    return _e(np.concatenate([spine, hori])), (h, w)


def _h_skeleton(m):
    N = 2 ** (m + 1) - 1
    edges = set()

    def seg(r0, c0, r1, c1):
        dr, dc = int(np.sign(r1 - r0)), int(np.sign(c1 - c0))
        r, c = r0, c0
        while (r, c) != (r1, c1):
            a, b = r * N + c, (r + dr) * N + c + dc
            edges.add((min(a, b), max(a, b)))
            r, c = r + dr, c + dc

    def rec(r, c, k):
        if k == 0:
            return
        d = 2 ** (k - 1)
        seg(r, c - d, r, c + d)
        seg(r - d, c - d, r + d, c - d)
        seg(r - d, c + d, r + d, c + d)
        for dr in (-d, d):
            for dc in (-d, d):
                rec(r + dr, c + dc, k - 1)

    rec(N // 2, N // 2, m)
    return N, sorted(edges)


def _flood(N, edges):
    """Attach every cell off the skeleton by a breadth-first flood from it (sources in id order, neighbours up, left,
    right, down): each new cell hangs from the cell that reached it."""
    on = np.zeros(N * N, bool)
    for a, b in edges:
        on[a] = on[b] = True
    queue = list(np.flatnonzero(on))
    out = list(edges)
    head = 0
    while head < len(queue):
        v = queue[head]
        head += 1
        r, c = divmod(int(v), N)
        for rr, cc in ((r - 1, c), (r, c - 1), (r, c + 1), (r + 1, c)):
            if 0 <= rr < N and 0 <= cc < N and not on[rr * N + cc]:
                on[rr * N + cc] = True
                out.append((int(v), rr * N + cc))
                queue.append(rr * N + cc)
    return out


def htree(m, widest=None):
    """H-tree of order m.  ``widest`` (from the centre root) sets the widest level, D deep, to exactly that many
    vertices by re-hanging leaves, which keeps a 4-connected grid tree: to trim, a leaf of level D moves onto a neighbour
    of level D + 1; to pad, a leaf of level D - 2 or D + 2 moves onto a neighbour of level D - 1.  (Grid neighbours
    differ in depth by an odd number, so a leaf cannot stay on its own level.)"""
    N, sk = _h_skeleton(m)
    edges = _flood(N, sk)
    if widest is not None:
        edges = _tune_widest(edges, N, widest)
    return _e(edges), (N, N)


def _tune_widest(edges, N, widest):
    root = (N // 2) * N + N // 2
    edges = {(min(a, b), max(a, b)) for a, b in edges}
    for _ in range(8):
        idx, par, _, lvl, L = canonical_bfs(_e(sorted(edges)), N * N, root)
        widths = np.diff(lvl)
        D = int(np.argmax(widths))
        excess = int(widths[D]) - widest
        if excess == 0:
            return sorted(edges)
        dv = np.empty(N * N, np.int64)
        dv[idx] = np.repeat(np.arange(L), widths)
        pv = np.empty(N * N, np.int64)
        pv[idx] = idx[par]
        pv[root] = -1
        deg = np.bincount(np.asarray(sorted(edges)).ravel(), minlength=N * N)
        sources = [D] if excess > 0 else [D - 2, D + 2]
        target = D + 1 if excess > 0 else D - 1
        moved = 0
        for s in sources:
            for v in idx[lvl[s]:lvl[s + 1]] if 0 <= s < L else []:
                if moved == abs(excess):
                    break
                if deg[v] != 1:
                    continue
                r, c = divmod(int(v), N)
                for rr, cc in ((r - 1, c), (r, c - 1), (r, c + 1), (r + 1, c)):
                    u = rr * N + cc
                    if 0 <= rr < N and 0 <= cc < N and u != pv[v] and dv[u] == target and deg[u] < 4:
                        edges.discard((min(v, pv[v]), max(v, pv[v])))
                        edges.add((min(u, v), max(u, v)))
                        deg[u] += 1
                        deg[pv[v]] -= 1
                        moved += 1
                        break
        if moved == 0:
            raise ValueError('cannot reach the requested widest level')
    raise ValueError('did not converge')


def broom(path_len, widths, seed=0):
    """Vertex 0 is the root; the path occupies levels 0 .. path_len - 1, then one level per entry of ``widths``."""
    rng = np.random.default_rng(seed)
    edges, prev = [], [0]
    for k in range(1, path_len):
        edges.append((k - 1, k))
        prev = [k]
    nxt = path_len
    for wdt in widths:
        cap = 4 if (prev == [0]) else 3
        assert wdt <= cap * len(prev), (wdt, len(prev))
        cur = list(range(nxt, nxt + wdt))
        nxt += wdt
        per = [wdt // len(prev) + (i < wdt % len(prev)) for i in range(len(prev))]
        k = 0
        for p, n in zip(prev, per):
            for _ in range(n):
                edges.append((p, cur[k]))
                k += 1
        prev = cur
    V = nxt
    perm = np.concatenate([[0], 1 + rng.permutation(V - 1)])       # vertex 0 stays the root
    e = perm[np.asarray(edges)]
    e = e[rng.permutation(len(e))]
    flip = rng.random(len(e)) < 0.5
    e[flip] = e[flip][:, ::-1]
    return _e(e), (1, V)


def grid_edges(h, w):
    v = np.arange(h * w).reshape(h, w)
    vert = np.stack([v[:-1, :], v[1:, :]], -1).reshape(-1, 2)
    hori = np.stack([v[:, :-1], v[:, 1:]], -1).reshape(-1, 2)
    return _e(np.concatenate([vert, hori]))


def random_mst(h, w, seed=0):
    from oracle.tree import mst_edge_ids
    ei = grid_edges(h, w)
    ew = np.random.default_rng(seed).random(len(ei)).astype(np.float32)
    return np.ascontiguousarray(ei[mst_edge_ids(ei, ew, h * w)]), (h, w)


def centre(hw):
    """TreeFilter2D._root: the centre pixel."""
    h, w = hw
    return (h // 2) * w + w // 2


# ---- canonical BFS ----
def canonical_bfs(edges, V, root=0):
    """The order bfs_forward promises, for any root: level by level, parents in position order, each vertex's children
    in ascending vertex id.  -> sorted_index [V], sorted_parent [V], sorted_child [V, 4] (positions, 0 = none),
    level_start [L + 1], L."""
    e = np.asarray(edges, dtype=np.int64)
    order = np.lexsort((np.concatenate([e[:, 1], e[:, 0]]), np.concatenate([e[:, 0], e[:, 1]])))
    src = np.concatenate([e[:, 0], e[:, 1]])[order]
    dst = np.concatenate([e[:, 1], e[:, 0]])[order]
    start = np.searchsorted(src, np.arange(V + 1))
    assert np.all(np.diff(start) <= 4), 'degree > 4'
    dst_l, start_l = dst.tolist(), start.tolist()
    idx = [root]
    pvert = [-1]
    par = [0]
    chd = np.zeros((V, 4), np.int32)
    lvl = [0, 1]
    ls, le = 0, 1
    while ls < le:
        for p in range(ls, le):
            v, pv = idx[p], pvert[p]
            k = 0
            for u in dst_l[start_l[v]:start_l[v + 1]]:
                if u == pv:
                    continue
                chd[p, k] = len(idx)
                k += 1
                idx.append(u)
                pvert.append(v)
                par.append(p)
        ls, le = le, len(idx)
        if le > ls:
            lvl.append(le)
    assert len(idx) == V, 'not a spanning tree'
    return (np.asarray(idx, np.int32), np.asarray(par, np.int32), chd, np.asarray(lvl, np.int32), len(lvl) - 1)


def profile(edges, V, root=0):
    """(L, widest level) from ``root``."""
    _, _, _, lvl, L = canonical_bfs(edges, V, root)
    return L, int(np.diff(lvl).max())


def dfs_order(edges, V, root=0):
    """A depth-first parent-before-child order of the same tree (children in DESCENDING vertex id): the kind of order
    the refine entry points must adopt.  -> sorted_index, sorted_parent, sorted_child (positions, 0 = none)."""
    e = np.asarray(edges, dtype=np.int64)
    adj = [[] for _ in range(V)]
    for a, b in e.tolist():
        adj[a].append(b)
        adj[b].append(a)
    out, par, pv = [], [], []
    stack = [(root, -1, 0)]
    while stack:
        v, p_vert, p_pos = stack.pop()
        out.append(v)
        par.append(p_pos)
        pv.append(p_vert)
        me = len(out) - 1
        for u in sorted(adj[v]):
            if u != p_vert:
                stack.append((u, v, me))
    idx = np.asarray(out, np.int32)
    par = np.asarray(par, np.int32)
    par[0] = 0
    chd = np.zeros((V, 4), np.int32)
    cnt = np.zeros(V, np.int64)
    for q in range(1, V):
        p = par[q]
        chd[p, cnt[p]] = q
        cnt[p] += 1
    return idx, par, chd


# ---- float64 refine over positions ----
def _tri(par, w):
    import scipy.sparse as sp
    V = len(par)
    rows = np.arange(1, V)
    # up:   U[p] - sum_{children c} w[c] U[c] = x[p]          (I - M) U = x,  M[par[c], c] = w[c]  (strictly upper)
    # down: A[p] - w[p] A[par[p]] = (1 - w[p]^2) U[p]         (I - N) A = D U, N[p, par[p]] = w[p] (strictly lower)
    eye = sp.identity(V, format='csr', dtype=np.float64)
    M = sp.csr_matrix((w[1:], (par[1:], rows)), shape=(V, V))
    N = sp.csr_matrix((w[1:], (rows, par[1:])), shape=(V, V))
    return (eye - M).tocsr(), (eye - N).tocsr()


def refine_f64(x, w, idx, par):
    """The refine recursion in float64, position by position (parents precede children, so one triangular solve per
    pass, no level loop):  U[p] = x[p] + sum_children w[c] U[c];  A[0] = U[0], A[p] = (1 - w[p]^2) U[p] + w[p] A[par];
    out = A / A(x = 1).  x [C, V] vertex-ordered, w [V] position-ordered (w[0] ignored) -> out [C, V] vertex-ordered."""
    from scipy.sparse.linalg import spsolve_triangular
    w = np.asarray(w, np.float64).copy()
    w[0] = 0.0
    par = np.asarray(par, np.int64)
    idx = np.asarray(idx, np.int64)
    up, down = _tri(par, w)
    xs = np.concatenate([np.asarray(x, np.float64)[:, idx], np.ones((1, len(idx)))]).T      # [V, C + 1]
    U = spsolve_triangular(up, xs, lower=False)
    A = spsolve_triangular(down, (1 - w * w)[:, None] * U, lower=True)
    out = np.empty((xs.shape[1] - 1, len(idx)))
    out[:, idx] = (A[:, :-1] / A[:, -1:]).T
    return out


def refine_f64_grad_feature(g, w, idx, par):
    """d <g, out> / d x for refine_f64 (the normaliser does not depend on x): the transposed solves, not the filter's
    symmetry.  g [C, V] vertex-ordered -> [C, V] vertex-ordered."""
    from scipy.sparse.linalg import spsolve_triangular
    w = np.asarray(w, np.float64).copy()
    w[0] = 0.0
    par = np.asarray(par, np.int64)
    idx = np.asarray(idx, np.int64)
    up, down = _tri(par, w)
    ones = np.ones((len(idx), 1))
    Z = spsolve_triangular(down, (1 - w * w)[:, None] * spsolve_triangular(up, ones, lower=False), lower=True)
    gs = np.asarray(g, np.float64)[:, idx].T / Z
    t = spsolve_triangular(down.T.tocsr(), gs, lower=False)
    gx = spsolve_triangular(up.T.tocsr(), (1 - w * w)[:, None] * t, lower=True)
    out = np.empty((gs.shape[1], len(idx)))
    out[:, idx] = gx.T
    return out


def edge_weight_f64(embed, idx, par, sigma):
    """embed [C, V] -> w [V] position-ordered: exp(-|E(v_p) - E(v_par)|^2 / sigma), w[0] = 0."""
    e = np.asarray(embed, np.float64)
    src = e[:, np.asarray(idx, np.int64)]
    d = src - src[:, np.asarray(par, np.int64)]
    w = np.exp(-(d * d).sum(0) / sigma)
    w[0] = 0.0
    return w


def grid_pitch(edges, V):
    """The row pitch bfs_grid_kernel infers (the largest non-unit |u - v| of an edge, V for a single row), or None when
    it rejects the tree as not 4-connected on that grid."""
    e = np.asarray(edges, np.int64)
    u, v = e.min(1), e.max(1)
    d = v - u
    nonunit = d[d != 1]
    wd = int(nonunit.max()) if len(nonunit) else V
    ok = (d > 0).all() and ((d == 1) | (d == wd)).all() and not ((d == 1) & (wd < V) & (v % wd == 0)).any()
    return wd if ok else None


# ---- the shapes the GPU tests run, with their level profile (L, widest level) from vertex 0 and from the centre ----
_BROOM_WIDE = [4, 12, 36, 108, 324]
SHAPES = {
    **{f'path1x{n}': (path, (n,)) for n in range(2, 9)},
    'path1x191489': (path, (GRID_BFS_MAX_V + 1,)),
    **{f'comb{h}x{w}': (comb, (h, w)) for h, w in [
        (33, 223), (33, 224), (33, 225), (129, 383), (129, 384), (129, 385), (129, 639), (129, 640), (129, 641),
        (33, 991), (33, 992), (33, 993), (257, 1023), (257, 1024), (257, 1025), (257, 200), (256, 748),
        (215, 244), (201, 261)]},
    **{f'serpentine{h}x{w}': (serpentine, (h, w)) for h, w in [(100, 100), (215, 244), (201, 261), (256, 748),
                                                                 (438, 438)]},
    'htree-m6': (htree, (6,)),
    'htree-m5-w1024': (htree, (5, 1024)),
    'htree-m5-w1025': (htree, (5, 1025)),
    'broom-L2-W4': (broom, (1, [4])),
    'broom-L6-W257': (broom, (1, [4, 12, 36, 108, 257])),
    **{f'broom-L7-W{w}': (broom, (1, _BROOM_WIDE + [w])) for w in (511, 512, 513)},
    'broom-L257-W1025': (broom, (250, [3, 9, 27, 81, 243, 729, 1025])),
    **{f'random{h}x{w}': (random_mst, (h, w)) for h, w in [(64, 80), (215, 244), (201, 261)]},
}
PROFILE = {          # name -> ((L, widest) from vertex 0, (L, widest) from the centre); checked by test_tree_shapes_cpu.py
    'path1x2': ((2, 1), (2, 1)), 'path1x3': ((3, 1), (2, 2)), 'path1x4': ((4, 1), (3, 2)), 'path1x5': ((5, 1), (3, 2)),
    'path1x6': ((6, 1), (4, 2)), 'path1x7': ((7, 1), (4, 2)), 'path1x8': ((8, 1), (5, 2)),
    'path1x191489': ((191489, 1), (95745, 2)),
    'comb33x223': ((255, 33), (350, 32)), 'comb33x224': ((256, 33), (352, 32)), 'comb33x225': ((257, 33), (353, 32)),
    'comb129x383': ((511, 129), (638, 128)), 'comb129x384': ((512, 129), (640, 128)),
    'comb129x385': ((513, 129), (641, 128)), 'comb129x639': ((767, 129), (1022, 128)),
    'comb129x640': ((768, 129), (1024, 128)), 'comb129x641': ((769, 129), (1025, 128)),
    'comb33x991': ((1023, 33), (1502, 32)), 'comb33x992': ((1024, 33), (1504, 32)), 'comb33x993': ((1025, 33), (1505, 32)),
    'comb257x1023': ((1279, 257), (1662, 256)), 'comb257x1024': ((1280, 257), (1664, 256)),
    'comb257x1025': ((1281, 257), (1665, 256)), 'comb257x200': ((456, 200), (428, 256)),
    'comb256x748': ((1003, 256), (1250, 255)), 'comb215x244': ((458, 215), (473, 214)),
    'comb201x261': ((461, 201), (491, 200)),
    'serpentine100x100': ((10000, 1), (5051, 2)), 'serpentine215x244': ((52460, 1), (26231, 2)),
    'serpentine201x261': ((52461, 1), (26231, 2)), 'serpentine256x748': ((191488, 1), (96119, 2)),
    'serpentine438x438': ((191844, 1), (96141, 2)),
    'htree-m6': ((255, 2408), (129, 4848)), 'htree-m5-w1024': ((127, 596), (65, 1024)),
    'htree-m5-w1025': ((127, 596), (65, 1025)),
    'broom-L2-W4': ((2, 4), (3, 3)), 'broom-L6-W257': ((6, 257), (10, 203)), 'broom-L7-W511': ((7, 511), (12, 405)),
    'broom-L7-W512': ((7, 512), (12, 431)), 'broom-L7-W513': ((7, 513), (12, 432)),
    'broom-L257-W1025': ((257, 1025), (255, 730)),
    'random64x80': ((363, 38), (233, 71)), 'random215x244': ((1619, 103), (1288, 114)),
    'random201x261': ((1272, 136), (1134, 136)),
}


_BUILT = {}


def build(name):
    """-> (edges, (h, w)) of SHAPES[name], built once per process."""
    if name not in _BUILT:
        fn, args = SHAPES[name]
        _BUILT[name] = fn(*args)
    return _BUILT[name]


def case_id(name, kind):
    """'<shape>-L<levels>-W<widest level>-<root>' for kind 'root0' (vertex 0) or 'centre' (TreeFilter2D._root)."""
    L, W = PROFILE[name][0 if kind == 'root0' else 1]
    return f'{name}-L{L}-W{W}-{kind}'


def root_vertex(name, kind):
    return 0 if kind == 'root0' else centre(build(name)[1])
