"""TEST INFRASTRUCTURE.  A plain restatement of the island-tile packing (k_tile_weights / k_tile_assign, DESIGN.md section 2)
and the checks that compare it with the packing the device reports (World.debug_tile_map).

An island (dynamic bodies with one label) is tiled when it has at most TILE_ISLAND_MAX dynamic bodies, manifolds with
points and joints, and at least one manifold or joint.  Its weight is the largest of the three counts.  Two-point islands
(no manifold with more than 2 points) and the others are packed separately, each in root-id order: with P the exclusive
prefix sum of the weights of its class and g = TILE_CAP + 1 - (heaviest tiled island of either class), an island goes
to tile P // g of its class; the two-point tiles come first.

Which islands are tiled changes only speed, never results, so nothing but a check like this one notices a packing that
sends every island to the dataflow path, puts one in the wrong class or overfills a tile."""
import numpy as np

TILE_CAP = 256
TILE_ISLAND_MAX = TILE_CAP // 2
TILE_NONE = 0xFFFFFFFF
SLOT_NONE = 0xFFFF
NO_ISLAND = 0xFFFFFFFF


def inputs(w, hinges):
    """What the packing depends on, as the host sees it after a step: island labels, which bodies are dynamic (awake),
    the manifolds with points (ordered body pairs, point counts) and the joints (body pairs)."""
    lab = w.islands()
    n = len(lab)
    dyn = lab != NO_ISLAND
    c = w.contacts()
    live = c["num"] > 0
    ha = np.asarray(hinges["a"], np.int64) if hinges else np.zeros(0, np.int64)
    hb = np.asarray(hinges["b"], np.int64) if hinges else np.zeros(0, np.int64)
    return dict(n=n, lab=lab, dyn=dyn, pairs=c["pairs"][live].astype(np.int64), num=c["num"][live].astype(np.int64), ha=ha, hb=hb)


def predict(x, max_tiles, multi_floor=None):
    """Restated packing of inputs `x`.  multi_floor: roots to count as multipoint whatever their manifolds say now (a
    generic tile's island keeps its tile while its manifolds drop to 2 points or fewer, until the next rebuild)."""
    n, lab, dyn = x["n"], x["lab"].astype(np.int64), x["dyn"]
    pa, pb = x["pairs"][:, 0], x["pairs"][:, 1]
    root_of_pair = np.where(dyn[pa], lab[pa], lab[pb])
    mdyn = dyn[pa] | dyn[pb]
    hdyn = dyn[x["ha"]] | dyn[x["hb"]]
    root_of_hinge = np.where(dyn[x["ha"]], lab[x["ha"]], lab[x["hb"]])
    nb = np.bincount(lab[dyn], minlength=n)
    nm = np.bincount(root_of_pair[mdyn], minlength=n)
    nh = np.bincount(root_of_hinge[hdyn], minlength=n)
    multi = np.zeros(n, bool)
    multi[root_of_pair[mdyn & (x["num"] > 2)]] = True
    if multi_floor is not None:
        multi |= multi_floor
    roots = np.nonzero(dyn & (lab == np.arange(n)))[0]
    ok = (nb[roots] <= TILE_ISLAND_MAX) & (nm[roots] <= TILE_ISLAND_MAX) & (nh[roots] <= TILE_ISLAND_MAX) & ((nm[roots] + nh[roots]) > 0)
    wgt = np.where(ok, np.maximum(nb[roots], np.maximum(nm[roots], nh[roots])), 0)
    wmax = int(wgt.max()) if len(wgt) else 0
    g = TILE_CAP + 1 - max(wmax, 1)
    two = ~multi[roots]
    p2 = np.cumsum(np.where(two, wgt, 0)) - np.where(two, wgt, 0)          # exclusive prefix sums in root order
    pg = np.cumsum(np.where(two, 0, wgt)) - np.where(two, 0, wgt)
    t2, tg = int(np.where(two, wgt, 0).sum()), int(np.where(two, 0, wgt).sum())
    ntiles2 = -(-t2 // g)
    ntiles = min(max_tiles, ntiles2 + -(-tg // g))
    tile_of_root = np.where(two, p2 // g, ntiles2 + pg // g)
    tile_of_root = np.where((wgt > 0) & (tile_of_root < max_tiles), tile_of_root, TILE_NONE)
    tile = np.full(n, TILE_NONE, np.int64)
    tile[roots] = tile_of_root
    return dict(roots=roots, nb=nb, nm=nm, nh=nh, multi=multi, weight=dict(zip(roots.tolist(), wgt.tolist())), wmax=wmax, g=g,
                ntiles2=min(max_tiles, ntiles2), ntiles=ntiles, tile=tile, root_of_pair=root_of_pair, mdyn=mdyn,
                root_of_hinge=root_of_hinge, hdyn=hdyn)


def check(m, x, p):
    """The device's map `m` (World.debug_tile_map) against the restatement `p` of inputs `x`; returns the number of
    bodies in tiles."""
    n, lab, dyn = x["n"], x["lab"].astype(np.int64), x["dyn"]
    assert m["ntiles"] == p["ntiles"] and m["ntiles2"] == p["ntiles2"], (m["ntiles"], m["ntiles2"], p["ntiles"], p["ntiles2"])
    want = np.where(dyn, p["tile"][np.where(dyn, lab, 0)], TILE_NONE)
    bad = np.nonzero(m["btile"].astype(np.int64) != want)[0]
    assert len(bad) == 0, f"{len(bad)} bodies in the wrong tile, e.g. body {bad[0]} (island {lab[bad[0]]}): tile {m['btile'][bad[0]]}, restated {want[bad[0]]}"
    assert (m["bslot"][~dyn | (want == TILE_NONE)] == SLOT_NONE).all()
    # the tiled constraints: [c0, c1) / [h0, h1) of each tile hold exactly those of its islands
    pkey = {tuple(q): k for k, q in enumerate(x["pairs"].tolist())}
    md, hd = p["mdyn"], p["hdyn"]
    tile_of_pair = np.where(md, p["tile"][np.where(md, p["root_of_pair"], 0)], TILE_NONE)
    tile_of_hinge = np.where(hd, p["tile"][np.where(hd, p["root_of_hinge"], 0)], TILE_NONE)
    assert m["ntiled"] == int((tile_of_pair != TILE_NONE).sum()), (m["ntiled"], int((tile_of_pair != TILE_NONE).sum()))
    assert m["nhtiled"] == int((tile_of_hinge != TILE_NONE).sum()), (m["nhtiled"], int((tile_of_hinge != TILE_NONE).sum()))
    covered_c, covered_h = 0, 0
    for t in range(m["ntiles"]):
        bodies = np.nonzero(m["btile"] == t)[0]
        nb = int(m["tile_nb"][t])
        assert nb == len(bodies) and nb <= TILE_CAP, (t, nb, len(bodies))      # ceil(total / g) tiles: the last may be empty
        assert np.array_equal(np.sort(m["bslot"][bodies]), np.arange(nb)), f"tile {t}: slots are not a permutation of [0, {nb})"
        c0, c1, h0, h1 = (int(m[k][t]) for k in ("tile_c0", "tile_c1", "tile_h0", "tile_h1"))
        assert c1 - c0 <= TILE_CAP and h1 - h0 <= TILE_CAP, (t, c0, c1, h0, h1)
        got = m["pairs"][c0:c1].tolist()
        assert len({tuple(q) for q in got}) == len(got)
        want_c = np.nonzero(tile_of_pair == t)[0]
        assert sorted(pkey.get(tuple(q), -1) for q in got) == want_c.tolist(), f"tile {t}: manifold range [{c0}, {c1}) is not its islands' manifolds"
        assert sorted(m["hinges"][h0:h1].tolist()) == np.nonzero(tile_of_hinge == t)[0].tolist(), f"tile {t}: hinge range [{h0}, {h1})"
        covered_c += c1 - c0; covered_h += h1 - h0
        if t < m["ntiles2"] and len(want_c):
            assert x["num"][want_c].max() <= 2, f"two-point tile {t} holds a manifold with {x['num'][want_c].max()} points"
    assert covered_c == m["ntiled"] and covered_h == m["nhtiled"]
    return int((want != TILE_NONE).sum())


class PackingCheck:
    """Per-step hook: checks the device's packing against the restatement on every step.  In CUDA-graph mode with the
    rebuild reuse, a step that skipped the rebuild must report the map of the last rebuilt step, and the inputs of the
    packing must not have changed since: the same manifolds with points, joints and dynamic bodies.  The one staleness
    allowed (DESIGN.md section 2) is a generic tile's island whose manifolds have all dropped to 2 points or fewer."""

    def __init__(self, scene):
        self.hinges = scene["hinges"]
        self.last = None            # (steps_rebuilt, map, inputs, multi) of the last rebuilt step
        self.rebuilt = self.reused = self.tiled_steps = 0
        self.history = []           # per step: tile of each island root, two-point tiles, (bodies, manifolds, joints) per tile

    def __call__(self, step, w):
        st = w.stats()
        m, x = w.debug_tile_map(), inputs(w, self.hinges)
        if self.last is not None and st["steps_rebuilt"] == self.last[0]:
            _, m0, x0, multi0 = self.last
            for k in ("btile", "bslot", "tile_nb", "tile_c0", "tile_c1", "tile_h0", "tile_h1", "pairs", "hinges"):
                assert np.array_equal(m[k], m0[k]), f"step {step}: reused rebuild, but the tile map's {k} changed"
            assert np.array_equal(x["dyn"], x0["dyn"]), f"step {step}: reused rebuild, but a body changed kind"
            assert {tuple(q) for q in x["pairs"].tolist()} == {tuple(q) for q in x0["pairs"].tolist()}, \
                f"step {step}: reused rebuild, but the set of manifolds with points changed"
            p = predict(x, m["max_tiles"], multi_floor=multi0)
            self.reused += 1
        else:
            p = predict(x, m["max_tiles"])
            self.last = (st["steps_rebuilt"], m, x, p["multi"])
            self.rebuilt += 1
        self.tiled_steps += check(m, x, p) > 0
        fill = np.stack([m["tile_nb"], m["tile_c1"] - m["tile_c0"], m["tile_h1"] - m["tile_h0"]], axis=1)
        md = p["mdyn"]
        dataflow = int((md & (p["tile"][np.where(md, p["root_of_pair"], 0)] == TILE_NONE)).sum())
        self.history.append(dict(tile=p["tile"], ntiles2=m["ntiles2"], fill=fill, weight=p["weight"], multi=p["multi"], dataflow=dataflow))
        return p
