"""Raycast on the GPU (include/b2d.h b2d_raycast): the device answer == the brute force (tests/raycast/ora_raycast.cpp) over every body, bit for
bit, on random worlds and on the four benchmark workloads at full size; the device-pointer path == the host-array path;
raycasts between steps change nothing the steps compute."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from tests import raycast_support as S  # noqa: E402
from tests.emu import raycast as R  # noqa: E402
from tests.parity import build_world, same_state  # noqa: E402


def _bounds(st, kind):
    dyn = np.asarray(kind) == 0
    bb = st["aabb"][:len(dyn)][dyn]
    return bb[:, :3].min(0), bb[:, 3:].max(0)


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_random_worlds_match_brute_force(gpu, E, seed):
    """Tilted static boxes, a plane, large bodies, bodies far outside the measured cell range, removed bodies, both ignore
    forms, zero-length and non-finite segments, segments cast right after add_bodies."""
    res = R.check_world(E, seed, n=400, rays=3000, steps=5)
    for x in res:
        assert x["mismatches"] == 0, x
    assert sum(x["hits"] for x in res) > 10000


def test_sleeping_bodies_are_candidates(gpu, E):
    """Boxes resting on a plane with island sleeping on: once they sleep, raycasts still see them."""
    scene = E.scenes.boxes_on_plane(3)
    w = E.scenes.build_world(scene, flags=E.world.FLAG_SLEEPING)
    for _ in range(20):
        w.step(60)
        if w.sleeping().sum() == len(scene["bodies"]["kind"]) - 1:
            break
    asleep = w.sleeping()
    assert asleep.sum() >= 20, asleep.sum()
    st = w.download_state()
    o = S.BruteWorld()
    o.add_bodies(scene["bodies"])
    o.set_state(st["pos"], st["orn"], st["linvel"], st["angvel"])
    p0, p1 = R.segments(np.random.default_rng(4), st["pos"], 2000, extent=3.0)
    g, c = w.raycast(p0, p1), o.raycast(p0, p1)
    assert R.compare(g, c)[1] == 0
    assert asleep[g["body"][g["body"] != E.RAY_MISS]].sum() > 200


WORKLOADS = {
    "boxes_4096": (lambda E: E.scenes.boxes_on_plane(16), 1 << 16, 2048),
    "spheres_65536": (lambda E: E.scenes.spheres_in_box(), 1 << 16, 1024),
    "mixed_262144": (lambda E: E.scenes.mixed_pile(64), 1 << 16, 512),
    "chains_1048576": (lambda E: E.scenes.hinge_chains(512, 512), 1 << 20, 192),
}


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_full_size_workloads_match_brute_force(gpu, E, name):
    """Each benchmark workload settled as bench.py does (150 steps), then a batch of mixed downward and horizontal
    segments; the brute force (loaded with the device state) checks a seeded sample of them."""
    make, nrays, nsample = WORKLOADS[name]
    scene = make(E)
    b = scene["bodies"]
    w = E.scenes.build_world(scene)
    w.step(150)
    st = w.download_state()
    lo, hi = _bounds(st, b["kind"])
    p0, p1 = E.scenes.raycast_segments(lo, hi, nrays, seed=3)
    g = w.raycast(p0, p1)
    assert (g["body"] != E.RAY_MISS).mean() > 0.3
    o = S.BruteWorld()
    o.add_bodies(b)
    o.set_state(st["pos"], st["orn"], st["linvel"], st["angvel"])
    pick = np.random.default_rng(5).choice(nrays, size=nsample, replace=False)
    c = o.raycast(p0[pick], p1[pick])
    sub = {k: v[pick] for k, v in g.items()}
    total, bad, first = R.compare(sub, c)
    assert bad == 0, (name, first, {k: v[first] for k, v in sub.items()}, {k: v[first] for k, v in c.items()})
    assert w.stats()["error_flags"] == 0


def test_device_pointer_path_equals_host_path(gpu, E):
    import torch
    scene = E.scenes.mixed_pile(16)
    w = E.scenes.build_world(scene)
    w.step(30)
    st = w.download_state()
    lo, hi = _bounds(st, scene["bodies"]["kind"])
    p0, p1 = E.scenes.raycast_segments(lo, hi, 50000, seed=1)
    ib = np.random.default_rng(2).integers(0, len(scene["bodies"]["kind"]), 50000).astype(np.uint32)
    ign = [0, 5, 17]
    host = w.raycast(p0, p1, ignore=ign, ignore_body=ib)
    dev = torch.device("cuda", 0)
    t0, t1 = torch.from_numpy(p0).to(dev), torch.from_numpy(p1).to(dev)
    tib = torch.from_numpy(ib.view(np.int32)).to(dev)
    body = torch.empty(50000, dtype=torch.int32, device=dev)
    frac = torch.empty(50000, dtype=torch.float32, device=dev)
    nrm = torch.empty((50000, 3), dtype=torch.float32, device=dev)
    feat = torch.empty(50000, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    w.raycast_device(50000, t0.data_ptr(), t1.data_ptr(), body.data_ptr(), frac.data_ptr(), nrm.data_ptr(), feat.data_ptr(),
                     ignore=ign, ignore_body_ptr=tib.data_ptr())
    w.sync()
    out = dict(body=body.cpu().numpy().view(np.uint32), fraction=frac.cpu().numpy(), normal=nrm.cpu().numpy(),
               feature=feat.cpu().numpy().view(np.uint32))
    assert R.compare(out, host)[1] == 0
    assert (host["body"] != E.RAY_MISS).sum() > 1000


@pytest.mark.parametrize("graph,reuse", [(True, True), (True, False), (False, True)])
def test_raycasts_do_not_change_stepping(gpu, E, graph, reuse):
    """200 steps with a raycast batch after every step == 200 steps without: state bits and rebuild counters."""
    scene = E.scenes.hinge_chains(16, 16, 4)
    env = dict(B2D_GRAPH="1" if graph else "0", B2D_GRAPH_REUSE="1" if reuse else "0")
    quiet, busy = build_world(E, scene, env=env), build_world(E, scene, env=env)
    busy.step(1)
    quiet.step(1)
    lo, hi = _bounds(busy.download_state(), scene["bodies"]["kind"])
    p0, p1 = E.scenes.raycast_segments(lo, hi, 4096, seed=0)
    hits = 0
    for s in range(199):
        quiet.step(1)
        busy.step(1)
        hits += int((busy.raycast(p0, p1)["body"] != E.RAY_MISS).sum())
        if s == 100:                                           # a disturbance: the island rebuild has to run again
            ids = np.arange(37 * 4, 38 * 4, dtype=np.uint32)
            up = np.tile(np.array([0.0, 3.0, 0.0], np.float32), (4, 1))
            for w in (quiet, busy):
                w.upload_bodies(ids, linvel=up)
    assert hits > 0
    same_state(quiet, busy)
    sa, sb = quiet.stats(), busy.stats()
    assert (sa["steps_rebuilt"], sa["steps_reused"]) == (sb["steps_rebuilt"], sb["steps_reused"])
    assert sb["error_flags"] == 0


def test_known_answers(gpu, E):
    """test/edyn/collision/test_raycast.cpp through the Python surface."""
    w = E.World(16)
    box = E.make_rigidbody(w, E.RigidBodyDef(kind=E.STATIC, shape=E.box_shape((0.5, 0.5, 0.5)), position=(0.5, 0.5, 0.5)))
    r = E.raycast(w, (2, 2, 2), (0, 0, 0))
    assert r.entity == box and r.fraction == 0.5 and r.info is not None
    r = E.raycast(w, (0.5, 2, 0.5), (0.5, 0, 0.5))
    assert r.entity == box and r.fraction == 0.5 and r.info == 2
    assert E.raycast(w, (0.5, 2, 0.5), (0.5, 0, 0.5), ignore_entities=[box]).entity is None
    assert E.raycast(w, (3, 3, 3), (4, 4, 4)).entity is None


CPP_KNOWN_ANSWERS = r"""
#include "edyn_adapter.hpp"
#include <cstdio>
int main() {
    edyn::registry registry;
    edyn::init_config cfg;
    cfg.max_bodies = 16; cfg.max_manifolds = 64;
    edyn::attach(registry, cfg);
    auto def = edyn::rigidbody_def{};
    def.kind = edyn::rigidbody_kind::rb_static;
    def.shape = edyn::box_shape{{0.5f, 0.5f, 0.5f}};
    def.position = {0.5f, 0.5f, 0.5f};
    auto box = edyn::make_rigidbody(registry, def);
    auto a = edyn::raycast(registry, {2, 2, 2}, {0, 0, 0});
    auto b = edyn::raycast(registry, {0.5f, 2, 0.5f}, {0.5f, 0, 0.5f});
    auto c = edyn::raycast(registry, {0.5f, 2, 0.5f}, {0.5f, 0, 0.5f}, {box});
    std::printf("%u %.9g %u %.9g %u %u\n", a.entity, a.fraction, b.entity, b.fraction, b.info, c.entity);
    edyn::detach(registry);
    return (a.entity == box && a.fraction == 0.5f && b.entity == box && b.fraction == 0.5f && b.info == 2 && c.entity == edyn::null) ? 0 : 1;
}
"""


def test_known_answers_cpp_adapter(gpu, tmp_path):
    """The same answers through edyn_adapter.hpp's edyn::raycast, compiled like hello_world.cpp."""
    import shutil
    import subprocess
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    src = tmp_path / "raycast_known.cpp"
    src.write_text(CPP_KNOWN_ANSWERS)
    exe = tmp_path / "raycast_known"
    libdir = os.path.join(ROOT, "edyn_b200")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(libdir, "csrc", "host"),
                        str(src), "-o", str(exe), "-L" + libdir, "-lb2d", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.stdout, r.stderr)


def test_golden_cases_as_one_batch(gpu, E):
    """Every non-plane case of tests/golden/raycast.npz as one world and one batch on the device == the reference's raw
    results through the filter rule, bit for bit (capsule hemisphere normals: == the brute force's corrected ones)."""
    from tests import test_raycast as T
    g = np.load(T.GOLDEN)
    sel = g["kind"] != T.PLANE
    soa = T.golden_world_soa(g, sel)
    w = E.World(len(soa["kind"]))
    w.add_bodies(soa)
    got = w.raycast(g["p0"][sel], g["p1"][sel])
    want = T.golden_expected(g, sel)
    o = S.BruteWorld()
    o.add_bodies(soa)
    hemi = (g["kind"][sel] == T.CAPSULE) & (want["feature"] <= 1)
    want["normal"][hemi] = o.raycast(g["p0"][sel], g["p1"][sel])["normal"][hemi]
    assert R.compare(got, want)[1] == 0
