"""The "empty ahead" table of build_empty_ahead (vpt_walk.cuh) restated in NumPy, checked against brute force over the node tables:

* every (node, child) entry and octant against a scan of all 512 leaves for a populated one in the orthant of the entry's block;
* the exactness argument itself: forward walks (p += d t, t >= 0, in float32, through the octree descent of oct_child) on octrees with
  uneven split planes never reach a populated leaf after passing an empty node whose entry says "nothing ahead";
* the fallback: a tree whose non-empty nodes split an axis at different floats for the same cell prefix gets an all-zero table."""
import numpy as np

AXIS_BIT = (1, 2, 4)


def upper(c, a):
    """upper-side bit of child c on axis a (the y bit of the child order means y-minus)"""
    return ((c >> 1) & 1) ^ 1 if a == 1 else (c >> (0 if a == 0 else 2)) & 1


def make_tree(occ, planes, root_min, root_max):
    """Node tables (pmin, half, pmax, child_empty) of the depth-3 octree over cell occupancy occ[x, y, z] whose split planes on axis a
    are planes[a] (9 sorted floats: box min, 7 splits, box max).  Empty internal nodes keep zeroed halves."""
    pmin = np.zeros((73, 3), np.float32); half = np.zeros((73, 3), np.float32); pmax = np.zeros((73, 3), np.float32)
    ce = np.zeros(73, np.uint32)

    def cells(path):                                   # cell ranges of the block at the end of the child path
        lo = [0, 0, 0]
        for l, c in enumerate(path):
            for a in range(3): lo[a] += upper(c, a) << (2 - l)
        n = 8 >> len(path)
        return [slice(lo[a], lo[a] + n) for a in range(3)], lo, n

    def fill(idx, path):
        sl, lo, n = cells(path)
        if not occ[tuple(sl)].any(): return                # empty: zeroed halves
        for a in range(3):
            pmin[idx, a] = planes[a][lo[a]]; pmax[idx, a] = planes[a][lo[a] + n]; half[idx, a] = planes[a][lo[a] + n // 2]
        for c in range(8):
            s2, _, _ = cells(path + [c])
            if not occ[tuple(s2)].any(): ce[idx] |= np.uint32(1 << c)

    fill(0, [])
    for c1 in range(8):
        fill(1 + c1, [c1])
        for c2 in range(8): fill(9 + c1 * 8 + c2, [c1, c2])
    return dict(pmin=pmin, half=half, pmax=pmax, ce=ce, root_min=np.float32(root_min), root_max=np.float32(root_max))


def full(t, i):
    re = int(t["ce"][0])
    if i < 9: return not (re >> (i - 1)) & 1
    c1, c2 = (i - 9) >> 3, (i - 9) & 7
    return not (re >> c1) & 1 and not (int(t["ce"][1 + c1]) >> c2) & 1


def leaf_populated(t):
    """[x, y, z] populated leaves, from child_empty bits alone (as the kernel reads them)"""
    re = int(t["ce"][0]); occ = np.zeros((8, 8, 8), bool)
    for c1 in range(8):
        if (re >> c1) & 1: continue
        for c2 in range(8):
            if (int(t["ce"][1 + c1]) >> c2) & 1: continue
            for c3 in range(8):
                if (int(t["ce"][9 + c1 * 8 + c2]) >> c3) & 1: continue
                occ[tuple(sum(upper(c, a) << (2 - l) for l, c in enumerate((c1, c2, c3))) for a in range(3))] = True
    return occ


def planes_consistent(t):
    for i in range(1, 73):
        if not full(t, i): continue
        l1 = i < 9
        c1, c2 = (i - 1, 0) if l1 else ((i - 9) >> 3, (i - 9) & 7)
        for a in range(3):
            free = 7 & ~AXIS_BIT[a]
            for m1 in range(8):
                for m2 in range(1 if l1 else 8):
                    if (m1 & ~free) or (m2 & ~free) or (m1 | m2) == 0: continue
                    j = 1 + (c1 ^ m1) if l1 else 9 + (c1 ^ m1) * 8 + (c2 ^ m2)
                    if full(t, j) and not t["half"][j, a] == t["half"][i, a]: return False
    return True


def entry_block(e):
    lvl = 1 if e < 8 else 2 if e < 72 else 3
    j = e if lvl == 1 else e - 8 if lvl == 2 else e - 72
    path = [j] if lvl == 1 else [j >> 3, j & 7] if lvl == 2 else [j >> 6, (j >> 3) & 7, j & 7]
    lo = [sum(upper(c, a) << (2 - l) for l, c in enumerate(path)) for a in range(3)]
    return lo, 8 >> lvl


def table_sweeps(t):
    """The kernel's construction: suffix-OR sweeps of the occupancy per octant, read at each block's first corner along the octant."""
    if not planes_consistent(t): return np.zeros((584, 8), bool)
    occ = leaf_populated(t)
    sfx = np.zeros((8, 8, 8, 8), bool)
    for o in range(8):
        s = occ.copy()
        for a in range(3):
            neg = (o >> a) & 1
            s = np.logical_or.accumulate(s, axis=a) if neg else np.flip(np.logical_or.accumulate(np.flip(s, a), axis=a), a)
        sfx[o] = s
    tab = np.zeros((584, 8), bool)
    for e in range(584):
        lo, n = entry_block(e)
        for o in range(8):
            cx, cy, cz = [lo[a] + n - 1 if (o >> a) & 1 else lo[a] for a in range(3)]
            tab[e, o] = not sfx[o, cx, cy, cz]
    return tab


def table_brute(t):
    occ = leaf_populated(t)
    pts = np.argwhere(occ)
    tab = np.zeros((584, 8), bool)
    for e in range(584):
        lo, n = entry_block(e)
        for o in range(8):
            ok = np.ones(len(pts), bool)
            for a in range(3):
                ok &= (pts[:, a] <= lo[a] + n - 1) if (o >> a) & 1 else (pts[:, a] >= lo[a])
            tab[e, o] = not ok.any()
    return tab


def random_tree(rs, density=0.08, even=False):
    occ = np.zeros((8, 8, 8), bool)
    for _ in range(rs.randint(1, 4)):                    # a few blobs of populated cells
        c = rs.randint(0, 8, 3); r = rs.randint(0, 3, 3)
        occ[max(c[0] - r[0], 0):c[0] + r[0] + 1, max(c[1] - r[1], 0):c[1] + r[1] + 1, max(c[2] - r[2], 0):c[2] + r[2] + 1] = True
    occ |= rs.rand(8, 8, 8) < density * 0.1
    lo = rs.uniform(-20, -5, 3).astype(np.float32); hi = rs.uniform(5, 20, 3).astype(np.float32)
    planes = []
    for a in range(3):
        inner = np.linspace(lo[a], hi[a], 9)[1:-1] if even else np.sort(rs.uniform(lo[a], hi[a], 7))
        planes.append(np.concatenate([[lo[a]], inner, [hi[a]]]).astype(np.float32))
    return make_tree(occ, planes, lo, hi)


def locate(t, p):
    """oct_locate_or_skip's descent: ('out'), ('leaf', index) or ('empty', entry)"""
    if not ((p >= t["root_min"]).all() and (p <= t["root_max"]).all()): return ("out", None)
    def child(i):
        h = t["half"][i]
        return int(not p[0] <= h[0]) + 2 * int(not p[1] >= h[1]) + 4 * int(not p[2] <= h[2])
    c1 = child(0)
    if (int(t["ce"][0]) >> c1) & 1: return ("empty", c1)
    c2 = child(1 + c1)
    if (int(t["ce"][1 + c1]) >> c2) & 1: return ("empty", 8 + c1 * 8 + c2)
    c3 = child(9 + c1 * 8 + c2)
    if (int(t["ce"][9 + c1 * 8 + c2]) >> c3) & 1: return ("empty", 72 + c1 * 64 + c2 * 8 + c3)
    return ("leaf", c1 * 64 + c2 * 8 + c3)


def test_table_matches_brute_force():
    rs = np.random.RandomState(3)
    n_ahead = 0
    for k in range(12):
        t = random_tree(rs, even=k % 2 == 0)
        assert planes_consistent(t)
        tab = table_sweeps(t)
        assert np.array_equal(tab, table_brute(t))
        n_ahead += int(tab.sum())
    assert n_ahead > 1000                                   # the trees have plenty of entries with nothing ahead


def test_forward_walks_never_meet_a_populated_leaf_after_an_empty_ahead_node():
    rs = np.random.RandomState(11)
    ended = 0
    for k in range(6):
        t = random_tree(rs, even=k % 2 == 0)
        tab = table_sweeps(t)
        lo, hi = t["root_min"], t["root_max"]
        for _ in range(1500):
            p = rs.uniform(lo, hi).astype(np.float32)
            d = rs.randn(3).astype(np.float32)
            d[rs.rand(3) < 0.1] = np.float32(0.0)            # axis-parallel rays: a zero component never moves
            if not d.any(): d[0] = np.float32(1.0)
            d = (d / np.linalg.norm(d)).astype(np.float32)
            o = int(d[0] < 0) | (int(d[1] < 0) << 1) | (int(d[2] < 0) << 2)
            armed = False
            for _ in range(400):
                kind, v = locate(t, p)
                if kind == "out": break
                if kind == "empty" and tab[v, o]: armed = True
                assert not (armed and kind == "leaf"), "a populated leaf after an empty-ahead node"
                # forward moves of every size the walks make: tiny steps, hops of at least 0.1, plane-snapping steps
                step = np.float32(rs.choice([rs.exponential(0.05), 0.1 + rs.exponential(1.0), 0.0]))
                p = (p + d * step).astype(np.float32)
            ended += armed
    assert ended > 1000


def test_split_planes_that_do_not_form_one_grid_give_an_empty_table():
    rs = np.random.RandomState(5)
    t = random_tree(rs, even=True)
    assert table_sweeps(t).any()
    # two non-empty level-2 nodes sharing their x cell prefix, one of them moved off the grid by one ulp
    nodes = [i for i in range(9, 73) if full(t, i)]
    pairs = [(i, j) for i in nodes for j in nodes if i < j and all(upper((i - 9) >> 3, 0) == upper((j - 9) >> 3, 0) for _ in [0])
             and upper((i - 9) & 7, 0) == upper((j - 9) & 7, 0)]
    assert pairs
    i, j = pairs[0]
    t["half"][j, 0] = np.nextafter(t["half"][j, 0], np.float32(np.inf))
    assert not planes_consistent(t)
    assert not table_sweeps(t).any()
    # the same change on an EMPTY node (its halves are never read) keeps the table
    t2 = random_tree(np.random.RandomState(5), even=True)
    empty = [i for i in range(9, 73) if not full(t2, i)]
    assert empty
    t2["half"][empty[0]] = np.float32(1.0)
    assert np.array_equal(table_sweeps(t2), table_brute(t2))
