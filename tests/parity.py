"""TEST INFRASTRUCTURE.  The device against the oracle in lock step (DESIGN.md section 6): one copy of the loops, the
oracle set-up and the comparisons every lock-step test makes, on the GPU or on the CPU emulation (tests/emu).

The oracle replays the device's Gauss-Seidel order (World.solver_order), so after each phase the two sides must agree:
ordered broadphase pairs as a multiset, with no unordered pair holding two manifolds; contact sets (counts,
attachments and lifetimes bit-equal, the 18 point floats within `tol`); island labels; the state within `tol`; hinge
impulses within `tol`.  Every comparison raises AssertionError naming the step and what differs, and is vectorised in
numpy, so it keeps up with the million-body worlds of tests/test_gpu_fullsize.py.

After a step the oracle continues from the device's state (`resync`), so every step is a fresh single-step comparison.
Whatever `resync` copies -- state, contacts with their warm-start impulses, hinge impulses -- it first compares with what
the oracle computed itself: a copy that nothing compared would hide a wrong value from every later step.

Nothing here imports edyn_b200 at module level: B2D_LIB (the emulation) has to be set before it is first imported."""
import hashlib
import os
import socket

import numpy as np

TOL = 1e-5
STATE_KEYS = ("pos", "orn", "linvel", "angvel", "aabb")

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


def check_contacts(step, gc, oc, tol=TOL):
    """Two contact sets (World.contacts / OracleWorld.contacts) matched by ordered pair: point counts, attachments and
    lifetimes bit-equal, the 18 floats of every point within `tol`."""
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
    err = np.abs(gc["pts"][gi][valid] - oc["pts"][oi][valid])
    if not err.max(initial=0) <= tol:
        raise AssertionError(f"step {step}: contact point floats differ by {err.max():.3e} (float {int(err.max(axis=0).argmax())})")


def same_partition(a, b):
    """Island labels are names, not values: two labelings describe the same partition iff the label pairs are in bijection."""
    pa = np.unique(np.stack([a.astype(np.int64), b.astype(np.int64)], 1), axis=0)
    return len(np.unique(pa[:, 0])) == len(pa) and len(np.unique(pa[:, 1])) == len(pa)


def check_islands(step, got, want, partition=False):
    """Island labels equal, or (partition) the same partition under other names."""
    if not (same_partition(got, want) if partition else np.array_equal(got, want)):
        raise AssertionError(f"step {step}: island {'partition' if partition else 'labels'} differ")


def check_state(step, got, want, tol=TOL, keys=STATE_KEYS, live=None):
    """Each of `keys` within `tol` over the bodies in `live` (default all); returns the largest difference per key."""
    errs = {k: float(np.abs(got[k] - want[k]).max(initial=0) if live is None else np.abs(got[k][live] - want[k][live]).max(initial=0))
            for k in keys}
    if not max(errs.values()) <= tol:
        raise AssertionError(f"step {step}: state differs: {errs}")
    return errs


def check_hinge_impulses(step, got, want, tol=TOL, alive=None):
    """The five impulses of every (live) hinge within `tol`."""
    err = np.abs(got - want) if alive is None else np.abs(got[alive] - want[alive])
    if not err.max(initial=0) <= tol:
        raise AssertionError(f"step {step}: hinge impulses differ by {err.max():.3e}")


def live_bodies(w):
    """The bodies the device has not removed (removed slots are not compared)."""
    return ~w.removed[:w.num_bodies]


def same_state(*worlds, keys=STATE_KEYS):
    """Every world's state bit-identical to the first's."""
    ref = worlds[0].download_state(aabb=True, inv_IW="inv_IW" in keys)
    for i, w in enumerate(worlds[1:], 1):
        check_state(f"world {i}", w.download_state(aabb=True, inv_IW="inv_IW" in keys), ref, tol=0.0, keys=keys)


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


def narrow(E, O, w, o, step, tol=TOL):
    """Both narrowphases; the contact sets compared."""
    w.run_phases(E.world.PH_NARROW); o.run_phases(O.PH_NARROW)
    check_contacts(step, w.contacts(), o.contacts(), tol)


def islands(E, O, w, o, step, partition=False):
    """Both island phases; the labels compared."""
    w.run_phases(E.world.PH_ISLANDS); o.run_phases(O.PH_ISLANDS)
    check_islands(step, w.islands(), o.islands(), partition)


def solve(E, O, w, o, step, tol=TOL):
    """The device's solve, then the oracle's with the device's order replayed; the live bodies' state compared.  Returns
    the device state and the largest difference per key."""
    w.run_phases(E.world.PH_SOLVE)
    hi, pr = w.solver_order()
    o.set_order(hi, pr)
    o.run_phases(O.PH_SOLVE)
    g = w.download_state(aabb=True)
    return g, check_state(step, g, o.state(), tol, live=live_bodies(w))


def resync(o, w, step, state, tol=TOL, compare_hinge_impulses=True):
    """Compare the device's contacts (with the impulses the solve stored for warm starting) and hinge impulses with the
    oracle's, then copy them and the device's `state` (already compared) into the oracle.  Returns the device's contacts."""
    gc = w.contacts()
    check_contacts(step, gc, o.contacts(), tol)
    if o.num_hinges and compare_hinge_impulses:
        check_hinge_impulses(step, w.hinge_impulses(), o.hinge_impulses(), tol, w.hinge_alive)
    load(o, w, state, gc)
    return gc


def phase_step(E, O, w, o, step, tol=TOL, partition=False, compare_hinge_impulses=True):
    """One step, phase by phase on both sides, everything compared, then the oracle resynchronised.  Returns the largest
    state difference per key."""
    broad(E, O, w, o, step)
    narrow(E, O, w, o, step, tol)
    islands(E, O, w, o, step, partition)
    g, errs = solve(E, O, w, o, step, tol)
    resync(o, w, step, g, tol, compare_hinge_impulses)
    return errs


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
    max_bodies reserves room for bodies added on the way.  Returns ok, worst (largest state difference), exact
    (bit-identical steps), points (contact points at the end), max_points (most points in one manifold at any step),
    flags, and digests: one hash of the device state and ordered pair set per step, for comparing modes.  On a
    difference: ok False, the step and why."""
    st = dict(scene["settings"])
    if vel_iters is not None:
        st["velocity_iterations"] = vel_iters
    if pos_iters is not None:
        st["position_iterations"] = pos_iters
    w = build_world(E, scene, mode, env, flags=E.world.FLAG_RESTITUTION_SOLVER if restitution_solver else 0, max_bodies=max_bodies, **st)
    o = oracle_for(O, scene, vel_iters=st["velocity_iterations"], pos_iters=st["position_iterations"], restitution=restitution_solver)
    worst, exact, max_points, digests = 0.0, 0, 0, []
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
                g = w.download_state(aabb=True)
                err = max(check_state(s, g, o.state(), live=live_bodies(w)).values())
                gc = resync(o, w, s, g)
            except AssertionError as e:
                return dict(ok=False, step=s, why=str(e))
            worst = max(worst, err)
            exact += err == 0.0
            digests.append(digest(g, wp))
            max_points = max(max_points, int(gc["num"].max(initial=0)))
            if hook is not None:
                hook(s, w)
        stats = w.stats()
    finally:
        w.close()
    return dict(ok=stats["error_flags"] == 0, worst=worst, exact=exact, points=int(stats["contact_points"]), max_points=max_points,
                flags=int(stats["error_flags"]), reused=int(stats["steps_reused"]), colors=int(stats["contact_colors"]), digests=digests)


def free_port():
    """A TCP port on 127.0.0.1 that was free a moment ago (for torch.distributed's rendezvous)."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p
