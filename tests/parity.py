"""TEST INFRASTRUCTURE.  The device against the oracle in lock step (DESIGN.md section 6): one copy of the loops, the
oracle set-up and the comparisons every lock-step test makes, on the GPU or on the CPU emulation (tests/emu).

The oracle replays the device's Gauss-Seidel order (World.solver_order), so after each phase the two sides must agree,
and they are compared as BITS (a float32 array viewed as uint32: -0 is not +0, a NaN equals nothing):
  * ordered broadphase pairs as a multiset, with no unordered pair holding two manifolds; island labels;
  * contact sets: counts, attachments, lifetimes and all 18 floats of every valid point;
  * linvel and angvel of every live body, and the hinge impulses;
  * the device's AABB and inverse world inertia of every live body against the oracle's refresh_body of the device's
    own pose;
  * pos and orn of every live body outside the TRIG SET (`trig_set`).
The one allowed difference is integrate()'s sinf / cosf (edyn_b200/csrc/b2d_math.cuh), which may differ from glibc's
by an ulp or two (tests/test_gpu_integrate.py pins by how much).  It runs after everything that writes a velocity or an
impulse, so only poses can differ: those of the bodies that took its sinf branch and of the rest of their islands
(the position iterations couple them), and with them the normal and distance the position iterations write back into
the contact points those bodies touch.  Inside the trig set pos / orn and those four point floats are held to
TRIG_TOL.  Under the CPU emulation (B2D_EMU=1) both sides call glibc and nothing is exempt.

After a step the oracle continues from the device's state (`resync`), so every step is a fresh single-step comparison.
Whatever `resync` copies -- state, contacts with their warm-start impulses, hinge impulses -- it first compares with what
the oracle computed itself: a copy that nothing compared would hide a wrong value from every later step.  Every
comparison raises AssertionError naming the step, what differs, the first offending body, pair or hinge and the
distance in ulps, and is vectorised in numpy, so it keeps up with the million-body worlds of tests/test_gpu_fullsize.py.

Nothing here imports edyn_b200 at module level: B2D_LIB (the emulation) has to be set before it is first imported."""
import hashlib
import os
import socket

import numpy as np

TRIG_TOL = 1e-5             # absolute, for the trig set's pos / orn and contact normal / distance only
TRIG_OMEGA = np.float32(0.001)       # integrate() takes its sinf branch at |w| >= 0.001f
TRIG_POINT_FLOATS = (6, 7, 8, 12)    # of the 18 point floats: normal (rewritten from the pose when attached) and distance
STATE_KEYS = ("pos", "orn", "linvel", "angvel", "aabb")
DYNAMIC, KINEMATIC, STATIC = 0, 1, 2
# How the device runs the step: plain launches that rebuild the islands every step, CUDA graphs that skip the rebuild while
# the constraint graph is unchanged, and everything on the dataflow path (no island tiles).  The emulation launches plainly.
MODES = {"plain": dict(B2D_GRAPH="0", B2D_GRAPH_REUSE="1", B2D_TILES="1"),
         "graph": dict(B2D_GRAPH="1", B2D_GRAPH_REUSE="1", B2D_TILES="1"),
         "dataflow": dict(B2D_GRAPH="0", B2D_GRAPH_REUSE="1", B2D_TILES="0")}


def build_world(E, scene, mode=None, env=None, **kw):
    """E.scenes.build_world with the environment of `mode` (read when the world is created) and the extra variables `env`;
    None: as the environment is."""
    env = {**(MODES[mode] if mode is not None else {}), **(env or {})}
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return E.scenes.build_world(scene, **kw)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def oracle_for(O, scene, *, vel_iters=None, pos_iters=None, threads=1, restitution=False, sleeping=False):
    """The oracle holding `scene`: bodies, hinges and exclusions, the scene's iteration counts unless overridden.
    restitution: the restitution solver at the reference's defaults (the device's conventions); sleeping: island sleeping."""
    st = scene["settings"]
    o = O.OracleWorld(vel_iters=st["velocity_iterations"] if vel_iters is None else vel_iters,
                      pos_iters=st["position_iterations"] if pos_iters is None else pos_iters, threads=threads)
    if restitution:
        o.set_restitution_iterations(8, 3)
    if sleeping:
        o.set_sleeping(True)
    o.add_bodies(scene["bodies"])
    if scene["hinges"]:
        h = scene["hinges"]
        o.add_hinges(h["a"], h["b"], h["pivot_a"], h["pivot_b"], h["axis_a"], h["axis_b"])
    if scene["exclusions"] is not None:
        o.add_exclusions(*scene["exclusions"])
    return o


def load(o, w, state=None, contacts=None):
    """Copy the device's state, contacts (with their warm-start impulses) and hinge impulses into the oracle, unchecked:
    for an oracle that starts from a state the device settled.  state / contacts: already downloaded."""
    g = w.download_state(aabb=False) if state is None else state
    c = w.contacts() if contacts is None else contacts
    o.set_state(g["pos"], g["orn"], g["linvel"], g["angvel"])
    o.set_contacts(c["pairs"], c["num"], c["pts"], c["att"], c["lifetime"])
    if o.num_hinges:
        o.set_hinge_impulses(w.hinge_impulses())


# ----------------------------------------------------------------------------- comparisons

def emulated():
    """The CPU emulation (B2D_EMU=1): glibc's sinf / cosf on both sides, so nothing is exempt from bit equality."""
    return os.environ.get("B2D_EMU") == "1"


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def ulps(a, b):
    """Distance in units in the last place between float32 values: the bit patterns laid on one monotone integer line,
    so -0 and +0 are one apart and a sign change counts every float in between."""
    def line(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF) - 1, i)
    return np.abs(line(a) - line(b))


def _first(step, what, got, want, bad, name):
    """The AssertionError for the bit differences `bad` (same shape as got / want, first axis the rows); name(row)
    says which body, pair or hinge a row is."""
    at = tuple(int(x) for x in np.argwhere(bad)[0])
    u = ulps(got[bad], want[bad])
    return AssertionError(f"step {step}: {what} differs in {int(bad.reshape(len(bad), -1).any(axis=1).sum())} of {len(bad)}; "
                          f"first at {name(at[0])}, component {at[1:]}: {got[at]!r} against {want[at]!r} ({int(ulps(got[at], want[at]))} ulp); "
                          f"largest {int(u.max())} ulp")


def check_bits(step, what, got, want, rows=None, label="body"):
    """got and want (float32, first axis the rows) bit-identical over `rows` (a boolean mask; default all).  Returns the
    number of rows compared."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    idx = np.arange(len(got)) if rows is None else np.nonzero(rows)[0]
    g, w = got[idx], want[idx]
    bad = _bits(g) != _bits(w)
    if bad.any():
        raise _first(step, what, g, w, bad, lambda r: f"{label} {int(idx[r])}")
    return len(idx)


def _keys(pairs):
    p = np.asarray(pairs, np.uint64).reshape(-1, 2)
    return (p[:, 0] << np.uint64(32)) | p[:, 1]


def check_pairs(step, got, want):
    """Ordered pairs (body[0], body[1]) equal as multisets, and no unordered pair in more than one manifold."""
    gk, wk = np.sort(_keys(got)), np.sort(_keys(want))
    if not np.array_equal(gk, wk):
        extra, missing = np.setdiff1d(gk, wk), np.setdiff1d(wk, gk)
        raise AssertionError(f"step {step}: ordered broadphase pair lists differ ({len(gk)} against {len(wk)}; "
                             f"{len(extra)} not expected, {len(missing)} missing)")
    p = np.asarray(got, np.uint64).reshape(-1, 2)
    u = np.unique((p.min(axis=1) << np.uint64(32)) | p.max(axis=1))
    if len(u) != len(p):
        raise AssertionError(f"step {step}: {len(p) - len(u)} pairs have more than one manifold")


def check_contacts(step, gc, oc, trig=None, tol=TRIG_TOL):
    """Two contact sets (World.contacts / OracleWorld.contacts) matched by ordered pair: point counts, attachments,
    lifetimes and the 18 floats of every point bit-equal.  trig: the trig set (`trig_set`); the normal and distance of
    the points of a manifold with a body in it are held to `tol` instead.  Returns the largest such difference."""
    gk, ok = _keys(gc["pairs"]), _keys(oc["pairs"])
    gi, oi = np.argsort(gk, kind="stable"), np.argsort(ok, kind="stable")
    if not np.array_equal(gk[gi], ok[oi]):
        raise AssertionError(f"step {step}: the manifolds' pairs differ ({len(gk)} against {len(ok)})")
    num = gc["num"][gi]
    bad = np.nonzero(num != oc["num"][oi])[0]
    if len(bad):
        raise AssertionError(f"step {step}: point counts differ for {len(bad)} manifolds, first {tuple(gc['pairs'][gi[bad[0]]])}: "
                             f"{num[bad[0]]} against {oc['num'][oi[bad[0]]]}")
    valid = np.arange(4)[None, :] < num[:, None]
    for k in ("att", "lifetime"):
        if not np.array_equal(gc[k][gi][valid], oc[k][oi][valid]):
            raise AssertionError(f"step {step}: contact {k} differs")
    pairs = gc["pairs"][gi]
    g, o = gc["pts"][gi], oc["pts"][oi]
    exact = np.repeat(valid[:, :, None], 18, axis=2)
    worst = 0.0
    if trig is not None and len(pairs):
        loose = exact.copy()
        loose[..., :] &= (trig[pairs[:, 0]] | trig[pairs[:, 1]])[:, None, None]
        loose[..., [k for k in range(18) if k not in TRIG_POINT_FLOATS]] = False
        exact &= ~loose
        if loose.any():
            worst = float(np.abs(g[loose] - o[loose]).max())
            if not worst <= tol:
                err = np.where(loose, np.abs(g - o), 0)
                at = np.unravel_index(int(np.argmax(err)), err.shape)
                raise AssertionError(f"step {step}: contact normal / distance of the trig set differ by {worst:.3e} > {tol:g} "
                                     f"(pair {tuple(int(x) for x in pairs[at[0]])}, slot {at[1]}, float {at[2]})")
    bad = exact & (_bits(g) != _bits(o))
    if bad.any():
        raise _first(step, "a contact point float (slot, float)", g, o, bad, lambda r: f"pair {tuple(int(x) for x in pairs[r])}")
    return worst


def same_partition(a, b):
    """Island labels are names, not values: two labelings describe the same partition iff the label pairs are in bijection."""
    pa = np.unique(np.stack([a.astype(np.int64), b.astype(np.int64)], 1), axis=0)
    return len(np.unique(pa[:, 0])) == len(pa) and len(np.unique(pa[:, 1])) == len(pa)


def check_islands(step, got, want, partition=False):
    """Island labels equal, or (partition) the same partition under other names."""
    if not (same_partition(got, want) if partition else np.array_equal(got, want)):
        raise AssertionError(f"step {step}: island {'partition' if partition else 'labels'} differ")


def check_hinge_impulses(step, got, want, alive=None):
    """The five impulses of every (live) hinge bit-equal."""
    check_bits(step, "hinge impulse", got, want, alive, label="hinge")


def live_bodies(w):
    """The bodies the device has not removed (removed slots are not compared)."""
    return ~w.removed[:w.num_bodies]


def body_kinds(w):
    """The kind of every body as the adapter created it.  A world holding bodies it has no definition of (handed over
    from a peer) counts all of them dynamic: the conservative side for `trig_set`."""
    try:
        return np.asarray(w.body_defs(np.arange(w.num_bodies))["kind"])
    except IndexError:
        return np.zeros(w.num_bodies, np.uint32)


def trig_set(w, state, contacts, kinds=None):
    """The bodies whose pose after this step may depend on integrate()'s sinf / cosf (DESIGN.md section 6):
      1. the live, awake dynamic and kinematic bodies whose |angvel| -- float32, as integrate() computes it -- is at
         least 0.001, the threshold of its sinf branch;
      2. closed over the step's position coupling: every body of such a dynamic body's island, and the islands of the
         dynamic bodies sharing a manifold with points, or a hinge, with such a kinematic body.
    state: the device state after the step (angvel bit-checked already); contacts: its contacts."""
    kind = body_kinds(w) if kinds is None else np.asarray(kinds)
    live = live_bodies(w)
    x, y, z = (np.ascontiguousarray(state["angvel"][:, i], np.float32) for i in range(3))
    spin = live & (kind != STATIC) & ~w.sleeping() & (np.sqrt((x * x + y * y) + z * z) >= TRIG_OMEGA)
    dyn = live & (kind != STATIC) & (kind != KINEMATIC)
    seeds, kin = spin & dyn, spin & (kind == KINEMATIC)
    if kin.any():
        edges = [np.asarray(contacts["pairs"])[np.asarray(contacts["num"]) > 0].reshape(-1, 2)]
        h = w.hinge_defs()
        if h is not None:
            edges.append(np.stack([h["a"], h["b"]], 1)[w.hinge_alive])
        e = np.concatenate(edges).astype(np.int64)
        for a, b in ((0, 1), (1, 0)):
            seeds[e[kin[e[:, a]] & dyn[e[:, b]], b]] = True
    lab = w.islands()
    return kin | (dyn & np.isin(lab, lab[seeds]))


def check_body_state(step, w, got, want, contacts, strict=None, tol=TRIG_TOL):
    """The state after the step: linvel and angvel of every live body bit-equal; pos and orn bit-equal outside the trig set
    and within `tol` inside it (strict, default under the emulation: bit-equal everywhere).  Stores the trig set in
    got["trig"] for `resync`.  Returns bitwise (dynamic and kinematic bodies outside the trig set: their poses compared
    bit for bit), trig (bodies in the trig set), worst (largest pose difference inside it) and exact (every pose
    bit-equal)."""
    live = live_bodies(w)
    for k in ("linvel", "angvel"):
        check_bits(step, k, got[k], want[k], live)
    kinds = body_kinds(w)
    trig = got["trig"] = trig_set(w, got, contacts, kinds)
    strict = emulated() if strict is None else strict
    bitwise = live if strict else live & ~trig
    for k in ("pos", "orn"):
        check_bits(step, k + (" (strict)" if strict else " outside the trig set"), got[k], want[k], bitwise)
    loose = live & trig
    worst = max(float(np.abs(got[k][loose] - want[k][loose]).max(initial=0)) for k in ("pos", "orn"))
    if not worst <= tol:
        raise AssertionError(f"step {step}: pos / orn of the trig set differ by {worst:.3e} > {tol:g}")
    exact = all(np.array_equal(_bits(got[k][loose]), _bits(want[k][loose])) for k in ("pos", "orn"))
    return dict(bitwise=int((bitwise & ~trig & (kinds != STATIC)).sum()), trig=int(loose.sum()), worst=worst, exact=exact)


def check_refresh(step, w, got, want):
    """The device's AABB and inverse world inertia of every live body bit-equal to the oracle's refresh_body of the
    device's own pose (want: the oracle's state after `load`)."""
    live = live_bodies(w)
    check_bits(step, "aabb (against the refresh of the device's pose)", got["aabb"], want["aabb"], live)
    check_bits(step, "inv_IW (against the refresh of the device's pose)", got["inv_IW"], want["inv_IW"], live)


def same_state(*worlds, keys=STATE_KEYS):
    """Every world's state bit-identical to the first's."""
    ref = worlds[0].download_state(aabb=True, inv_IW="inv_IW" in keys)
    for i, w in enumerate(worlds[1:], 1):
        g = w.download_state(aabb=True, inv_IW="inv_IW" in keys)
        for k in keys:
            check_bits(f"world {i}", k, g[k], ref[k])


def same_digests(runs):
    """runs: {name: one digest per step}.  Every run bit-identical to the first, step by step."""
    (first, ref), *rest = runs.items()
    for name, d in rest:
        diff = [s for s, (a, b) in enumerate(zip(ref, d)) if a != b]
        assert not diff and len(d) == len(ref), f"{name} differs from {first} from step {diff[0] if diff else min(len(d), len(ref))} on"


def digest(state, pairs):
    """One hash of the device state and its ordered pair set."""
    p = pairs[np.lexsort((pairs[:, 1], pairs[:, 0]))] if len(pairs) else pairs
    return hashlib.sha1(b"".join(np.ascontiguousarray(x).tobytes() for x in [state[k] for k in STATE_KEYS] + [p])).hexdigest()


# ----------------------------------------------------------------------------- the phases, one at a time

def broad(E, O, w, o, step):
    """Both broadphases; the pair lists compared.  Returns the device's pairs."""
    w.run_phases(E.world.PH_BROAD); o.run_phases(O.PH_BROAD)
    got = w.pairs()
    check_pairs(step, got, o.pairs())
    return got


def narrow(E, O, w, o, step):
    """Both narrowphases; the contact sets compared bit for bit (no pose has been integrated yet)."""
    w.run_phases(E.world.PH_NARROW); o.run_phases(O.PH_NARROW)
    check_contacts(step, w.contacts(), o.contacts())


def islands(E, O, w, o, step, partition=False):
    """Both island phases; the labels compared."""
    w.run_phases(E.world.PH_ISLANDS); o.run_phases(O.PH_ISLANDS)
    check_islands(step, w.islands(), o.islands(), partition)


def solve(E, O, w, o, step, strict=None):
    """The device's solve, then the oracle's with the device's order replayed; the live bodies' state compared
    (`check_body_state`).  Returns the device state (with its trig set) and the report of `check_body_state`."""
    w.run_phases(E.world.PH_SOLVE)
    hi, pr = w.solver_order()
    o.set_order(hi, pr)
    o.run_phases(O.PH_SOLVE)
    g = w.download_state(aabb=True, inv_IW=True)
    return g, check_body_state(step, w, g, o.state(), w.contacts(), strict)


def resync(o, w, step, state, compare_hinge_impulses=True, contacts=None, strict=None):
    """Compare the device's contacts (with the impulses the solve stored for warm starting) and hinge impulses with the
    oracle's, then copy them and the device's `state` (already compared) into the oracle, and compare the device's AABBs
    and inverse world inertias with the oracle's refresh of that state.  state: from `solve` or `check_body_state` (its
    trig set is computed here otherwise); contacts: the device's, if downloaded already.  Returns the device's contacts
    and the largest difference of the trig set's contact normals and distances."""
    gc = w.contacts() if contacts is None else contacts
    trig = state["trig"] if "trig" in state else trig_set(w, state, gc)
    worst = check_contacts(step, gc, o.contacts(), None if (emulated() if strict is None else strict) else trig)
    if o.num_hinges and compare_hinge_impulses:
        check_hinge_impulses(step, w.hinge_impulses(), o.hinge_impulses(), w.hinge_alive)
    load(o, w, state, gc)
    check_refresh(step, w, state if "inv_IW" in state and "aabb" in state else w.download_state(aabb=True, inv_IW=True), o.state())
    return gc, worst


def phase_step(E, O, w, o, step, partition=False, compare_hinge_impulses=True):
    """One step, phase by phase on both sides, everything compared, then the oracle resynchronised.  Returns the report of
    `check_body_state`, its worst and exact covering the trig set's contact floats too."""
    broad(E, O, w, o, step)
    narrow(E, O, w, o, step)
    islands(E, O, w, o, step, partition)
    g, rep = solve(E, O, w, o, step)
    _, cworst = resync(o, w, step, g, compare_hinge_impulses)
    rep["exact"] = rep["exact"] and cworst == 0.0
    rep["worst"] = max(rep["worst"], cworst)
    return rep


def tally(res, rep):
    """A run's total (None: none yet) with one more step's report of `phase_step` added."""
    res = res or dict(bitwise=0, trig=0, worst=0.0, exact=0)
    return dict(bitwise=res["bitwise"] + rep["bitwise"], trig=res["trig"] + rep["trig"], worst=max(res["worst"], rep["worst"]),
                exact=res["exact"] + rep["exact"])


def report(name, res):
    """Print one line for the test log: body-steps whose pose was compared bit for bit, body-steps in the trig set, the
    largest difference inside it and the bit-identical steps (pytest -rP shows it)."""
    n = res["bitwise"] + res["trig"]
    print(f"parity {name}: {res['bitwise']} body-steps bitwise, {res['trig']} in the trig set "
          f"({res['trig'] / max(n, 1):.1%}), largest trig-set difference {res['worst']:.2e}, {res['exact']} bit-identical steps")


def oracle_step(O, o, w):
    """The oracle's whole step with the order of the device's last step replayed (the device has stepped already)."""
    hi, pr = w.solver_order()
    o.run_phases(O.PH_BROAD | O.PH_NARROW | O.PH_ISLANDS)
    o.set_order(hi, pr)
    o.run_phases(O.PH_SOLVE)


# ----------------------------------------------------------------------------- whole steps

def lockstep(E, O, scene, steps, restitution_solver=False, mode=None, hook=None, vel_iters=None, pos_iters=None, env=None,
             before=None, max_bodies=None):
    """One device world in `mode` (a key of MODES; None: as the environment says) against the oracle, `steps` whole
    steps (World.step), each compared after the step: pairs, island labels, state, then contacts and hinge impulses as
    `resync` copies them.  vel_iters / pos_iters override the scene's settings on both sides; env: more environment
    variables for the world's creation; hook(step, world) runs after each step's comparison (and may assert);
    before(step, world, oracle) runs before each step, may change both worlds and returns the oracle to continue with;
    max_bodies reserves room for bodies added on the way.  Returns ok; bitwise (body-steps whose pose was compared bit
    for bit); trig (body-steps in the trig set); worst (largest difference inside the trig set); exact (steps bit-identical
    throughout, the trig set included); points (contact points at the end); max_points (most points in one manifold at
    any step); flags; and digests: one hash of the device state and ordered pair set per step, for comparing modes.  On
    a difference: ok False, the step and why."""
    st = dict(scene["settings"])
    if vel_iters is not None:
        st["velocity_iterations"] = vel_iters
    if pos_iters is not None:
        st["position_iterations"] = pos_iters
    w = build_world(E, scene, mode, env, flags=E.world.FLAG_RESTITUTION_SOLVER if restitution_solver else 0, max_bodies=max_bodies, **st)
    o = oracle_for(O, scene, vel_iters=st["velocity_iterations"], pos_iters=st["position_iterations"], restitution=restitution_solver)
    worst, exact, bitwise, trig, max_points, digests = 0.0, 0, 0, 0, 0, []
    try:
        for s in range(steps):
            if before is not None:
                o = before(s, w, o)
            w.step(1)
            oracle_step(O, o, w)
            try:
                wp = w.pairs()
                check_pairs(s, wp, o.pairs())
                check_islands(s, w.islands(), o.islands())
                g = w.download_state(aabb=True, inv_IW=True)
                gc = w.contacts()
                rep = check_body_state(s, w, g, o.state(), gc)
                _, cworst = resync(o, w, s, g, contacts=gc)
            except AssertionError as e:
                return dict(ok=False, step=s, why=str(e))
            worst = max(worst, rep["worst"], cworst)
            exact += rep["exact"] and cworst == 0.0
            bitwise += rep["bitwise"]
            trig += rep["trig"]
            digests.append(digest(g, wp))
            max_points = max(max_points, int(gc["num"].max(initial=0)))
            if hook is not None:
                hook(s, w)
        stats = w.stats()
    finally:
        w.close()
    return dict(ok=stats["error_flags"] == 0, worst=worst, exact=exact, bitwise=bitwise, trig=trig, points=int(stats["contact_points"]),
                max_points=max_points, flags=int(stats["error_flags"]), reused=int(stats["steps_reused"]), colors=int(stats["contact_colors"]),
                digests=digests)


def free_port():
    """A TCP port on 127.0.0.1 that was free a moment ago (for torch.distributed's rendezvous)."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p
