"""The N > 1 path on CPU: island-aware partitioning, sub-scene extraction and the per-step bounds exchange, with a real
two-process torch.distributed group on the gloo backend (127.0.0.1)."""
import os

import numpy as np
import pytest

from tests.parity import free_port

f32 = np.float32


def test_partition_keeps_islands_whole(E):
    from edyn_b200 import dist
    scene = E.scenes.hinge_chains(6, 4)
    lab = dist.initial_islands(scene)
    n = scene["dynamic"]
    chains = lab[:n].reshape(-1, 4)
    assert (chains == chains[:, :1]).all(), "a chain is one island"
    assert len(np.unique(chains[:, 0])) == 24
    for ws in (2, 3, 4):
        owner = dist.partition(scene, ws, lab)
        assert (owner[n:] == -1).all(), "static bodies are replicated"
        assert set(np.unique(owner[:n])) == set(range(ws))
        o = owner[:n].reshape(-1, 4)
        assert (o == o[:, :1]).all(), "an island never straddles two ranks"
        counts = np.bincount(owner[:n], minlength=ws)
        assert counts.max() - counts.min() <= 8
        parts = [dist.shard(scene, r, ws, owner) for r in range(ws)]
        assert sum(p["dynamic"] for p in parts) == n
        gids = np.concatenate([p["global_ids"][p["bodies"]["kind"] == 0] for p in parts])
        assert len(np.unique(gids)) == n, "every dynamic body is owned by exactly one rank"
        for p in parts:
            h = p["hinges"]
            assert h is not None and (h["b"] - h["a"] == 1).all() and h["b"].max() < len(p["bodies"]["kind"])
            assert len(h["a"]) == 3 * p["dynamic"] // 4
            ea, eb = p["exclusions"]
            assert len(ea) == len(h["a"])


def test_initial_islands_follow_aabb_proximity(E):
    from edyn_b200 import dist
    scene = E.scenes.boxes_on_plane(3)          # 27 unit boxes at 1.1 pitch
    lab = dist.initial_islands(scene)
    n = scene["dynamic"]
    assert len(np.unique(lab[:n])) == 27        # 0.1 gaps in every direction at t = 0: nothing within the 0.026 margin
    lab = dist.initial_islands(scene, reach=0.25)
    assert len(np.unique(lab[:n])) == 1


def test_overlapping_ranks():
    from edyn_b200 import dist
    b = np.array([[0, 0, 0, 1, 1, 1], [1.01, 0, 0, 2, 1, 1], [5, 5, 5, 6, 6, 6], [np.nan] * 6], f32)
    assert dist.overlapping_ranks(b) == [(0, 1)]
    assert dist.overlapping_ranks(b, margin=0.001) == []


def _worker(rank, world_size, port, q):
    import torch.distributed as dist_mod
    import edyn_b200 as E
    from edyn_b200 import dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist_mod.init_process_group("gloo", rank=rank, world_size=world_size)
    try:
        scene = E.scenes.hinge_chains(4, 2)
        owner = dist.partition(scene, world_size)
        local = dist.shard(scene, rank, world_size, owner)
        # stand-in for ShardedWorld without a GPU: same exchange code path, bounds computed from the initial positions
        sw = dist.ShardedWorld.__new__(dist.ShardedWorld)
        sw.rank, sw.world_size, sw.dist, sw.local = rank, world_size, dist_mod, local
        sw.dynamic_local = np.where(local["bodies"]["kind"] == 0)[0]
        pos = local["bodies"]["pos"]
        aabb = np.concatenate([pos - 0.35, pos + 0.35], axis=1).astype(f32)
        far = sw.exchange_bounds(sw.local_bounds(aabb))
        hits_far = dist.overlapping_ranks(far)
        # now pretend rank 1's islands drifted into rank 0's region
        if rank == 1:
            aabb[:, [0, 3]] -= aabb[sw.dynamic_local][:, 0].min() - 1.0
        near = sw.exchange_bounds(sw.local_bounds(aabb))
        q.put((rank, local["dynamic"], far.tolist(), hits_far, dist.overlapping_ranks(near)))
    finally:
        dist_mod.destroy_process_group()


def test_bounds_exchange_gloo_world_size_2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (r0, n0, far0, hf0, hn0), (r1, n1, far1, hf1, hn1) = res
    assert n0 + n1 == 32 and n0 == n1 == 16
    assert far0 == far1, "all ranks see the same gathered bounds"
    assert hf0 == hf1 == [], "disjoint shards: no cross-rank overlap"
    assert hn0 == hn1 == [(0, 1)], "the drifted shard is detected on every rank"


def _migration_worker(rank, world_size, port, q):
    import torch.distributed as dist_mod
    import edyn_b200 as E
    from edyn_b200 import dist
    from tests._oracle_world import OracleBackedWorld
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist_mod.init_process_group("gloo", rank=rank, world_size=world_size)
    try:
        scene = E.scenes.approaching_stacks(height=2, gap=0.6, speed=3.0)
        sw = dist.ShardedWorld(scene, rank, world_size, dist_mod, world_factory=OracleBackedWorld)
        owned0 = len(sw.dynamic_local)
        first_hit = None
        for k in range(40):
            pairs = sw.step(1)
            if pairs and first_hit is None:
                first_hit = k
        st = sw.world.download_state()
        gids = np.asarray(sw.global_of_local)[sw.dynamic_local]
        q.put((rank, owned0, first_hit, sw.migrated_in, sw.migrated_out, gids.tolist(), st["pos"][sw.dynamic_local].tolist(),
               len(sw.world.contacts()["pairs"])))
    finally:
        dist_mod.destroy_process_group()


def test_island_migration_gloo_world_size_2(E):
    """Two stacks owned by two ranks slide into each other: the higher rank hands its island over, and the merged
    simulation on rank 0 tracks the single-world run of the same scene."""
    import torch.multiprocessing as mp
    from tests._oracle_world import OracleBackedWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_migration_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, own0, hit0, in0, out0, gid0, pos0, nc0), (_, own1, hit1, in1, out1, gid1, pos1, nc1) = res
    assert own0 == own1 == 2
    assert hit0 == hit1 and hit0 is not None and hit0 > 0, "both ranks see the overlap on the same step"
    assert (in0, out0, in1, out1) == (2, 0, 0, 2), "rank 1's island moved to rank 0, nothing else moved"
    assert sorted(gid0) == [0, 1, 2, 3] and gid1 == [] and nc1 == 0
    assert nc0 >= 4, "ground contacts of both stacks plus the stack-stack contacts live on rank 0"
    # single-world run of the same scene (same oracle): same bodies by global id
    scene = E.scenes.approaching_stacks(height=2, gap=0.6, speed=3.0)
    ref = OracleBackedWorld(scene)
    ref.step(40)
    want = ref.download_state()["pos"][:4]
    got = np.zeros((4, 3), f32)
    got[np.asarray(gid0)] = np.asarray(pos0, f32)
    # body ids (hence pair and Gauss-Seidel order) differ after the move, so the runs agree to solver tolerance, not bitwise
    assert np.abs(got - want).max() < 2e-3, np.abs(got - want).max()
    assert np.abs(got[:, 0].mean() - want[:, 0].mean()) < 1e-3


def _chain_migration_worker(rank, world_size, port, q):
    import torch.distributed as dist_mod
    import edyn_b200 as E
    from edyn_b200 import dist
    from tests._oracle_world import OracleBackedWorld
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist_mod.init_process_group("gloo", rank=rank, world_size=world_size)
    try:
        scene = E.scenes.hinge_chains(2, 2, 4)
        sw = dist.ShardedWorld(scene, rank, world_size, dist_mod, world_factory=OracleBackedWorld)
        sw.world.step(10)
        st = sw.world.download_state()
        bounds = sw.exchange_bounds(sw.local_bounds(st["aabb"]))
        assert dist.overlapping_ranks(bounds) == [], "the two chain groups are 3.5 m apart"
        # force the hand-over: pretend rank 0's islands have grown over everything
        if rank == 0:
            real = sw.island_boxes
            def grown(state):
                ids, box = real(state)
                return ids, box + np.array([-10, -10, -10, 10, 10, 10], f32)
            sw.island_boxes = grown
        sw.migrate([(0, 1)], bounds, st)
        sw.world.step(20)
        st = sw.world.download_state()
        gids = np.asarray(sw.global_of_local)[sw.dynamic_local]
        h = sw.world.hinge_defs()
        alive = int(sw.world.hinge_alive.sum()) if h is not None else 0
        q.put((rank, sw.migrated_in, sw.migrated_out, gids.tolist(), st["pos"][sw.dynamic_local].tolist(), alive,
               len(sw.world.exclusions), sorted(map(tuple, sw.world.o.pairs().tolist()))))
    finally:
        dist_mod.destroy_process_group()


def test_chain_islands_migrate_with_joints_and_exclusions(E):
    """Hinge chains change rank: the joints and the collision exclusions between adjacent links travel with the bodies
    (otherwise neighbouring links would start colliding on the new rank), and the result equals the single-world run."""
    import torch.multiprocessing as mp
    from tests._oracle_world import OracleBackedWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_chain_migration_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, in0, out0, gid0, pos0, h0, x0, pairs0), (_, in1, out1, gid1, pos1, h1, x1, pairs1) = res
    assert (in0, out0, in1, out1) == (8, 0, 0, 8)
    assert sorted(gid0) == list(range(16)) and gid1 == []
    assert h0 == 12 and h1 == 0, "3 joints per chain, all alive on rank 0, none left on rank 1"
    assert x0 == 12, "one exclusion per joint travelled along"
    scene = E.scenes.hinge_chains(2, 2, 4)
    ref = OracleBackedWorld(scene)
    ref.step(30)
    want = ref.download_state()["pos"][:16]
    got = np.zeros((16, 3), f32)
    got[np.asarray(gid0)] = np.asarray(pos0, f32)
    assert np.abs(got - want).max() < 1e-5, np.abs(got - want).max()
    # same number of manifolds as the single world: adjacent links are excluded on the new rank too
    ref_pairs = {tuple(p) for p in ref.o.pairs().tolist()}
    assert len(pairs0) == len(ref_pairs), (len(pairs0), len(ref_pairs))


def _interleaved_worker(rank, world_size, port, q):
    import torch.distributed as dist_mod
    import edyn_b200 as E
    from edyn_b200 import dist
    from tests._oracle_world import OracleBackedWorld
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist_mod.init_process_group("gloo", rank=rank, world_size=world_size)
    try:
        scene = E.scenes.hinge_chains(2, 8, 2)                  # 16 two-link chains, 0.5 m apart in z
        n = scene["dynamic"]
        owner = np.full(len(scene["bodies"]["kind"]), -1, np.int64)
        owner[:n] = (np.arange(n) // 2) % 2                      # neighbouring chains alternate between the ranks
        sw = dist.ShardedWorld(scene, rank, world_size, dist_mod, world_factory=OracleBackedWorld, owner=owner)
        flagged = 0
        for _ in range(15):
            flagged += bool(sw.step(1))
        q.put((rank, flagged, sw.migrated_in, sw.migrated_out, len(sw.dynamic_local)))
    finally:
        dist_mod.destroy_process_group()


def test_interleaved_ranks_do_not_migrate_without_island_contact():
    """Two ranks whose regions interleave (rank boxes overlap every step) keep their islands as long as no island of
    one comes within the broadphase margin of an island of the other: the decision is taken on island AABBs."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_interleaved_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, flagged, mig_in, mig_out, owned in res:
        assert flagged == 15, "the coarse rank-box test fires every step"
        assert mig_in == mig_out == 0 and owned == 16, "but no island actually touches one of the other rank"


def _three_rank_worker(rank, world_size, port, q):
    import torch.distributed as dist_mod
    import edyn_b200 as E
    from edyn_b200 import dist
    from tests._oracle_world import OracleBackedWorld
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist_mod.init_process_group("gloo", rank=rank, world_size=world_size)
    try:
        scene = E.scenes.hinge_chains(3, 2, 2)                  # 6 two-link chains in three x-slabs
        sw = dist.ShardedWorld(scene, rank, world_size, dist_mod, world_factory=OracleBackedWorld)
        owned0 = len(sw.dynamic_local)
        sw.world.step(5)
        st = sw.world.download_state()
        bounds = sw.exchange_bounds(sw.local_bounds(st["aabb"]))
        real = sw.island_boxes
        if rank < 2:                                             # ranks 0 and 1 pretend to have grown over everything
            sw.island_boxes = lambda state: (real(state)[0], real(state)[1] + np.array([-20, -20, -20, 20, 20, 20], f32))
        sw.migrate([(0, 1), (0, 2), (1, 2)], bounds, st)
        sw.world.step(5)
        gids = np.asarray(sw.global_of_local)[sw.dynamic_local]
        q.put((rank, owned0, sw.migrated_in, sw.migrated_out, sorted(gids.tolist())))
    finally:
        dist_mod.destroy_process_group()


def test_three_ranks_lowest_destination_wins():
    """A rank that touches two lower ranks hands each island over once, to the lowest of them; a rank that is both a
    destination and a source in the same exchange ends up consistent."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_three_rank_worker, args=(r, 3, port, q)) for r in range(3)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=240) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, o0, in0, out0, g0), (_, o1, in1, out1, g1), (_, o2, in2, out2, g2) = res
    assert o0 == o1 == o2 == 4
    assert (in0, out0) == (8, 0) and g0 == list(range(12)), "everything ends up on rank 0"
    assert (in1, out1) == (0, 4) and g1 == [], "rank 1 gave its islands to rank 0 and received none from rank 2"
    assert (in2, out2) == (0, 4) and g2 == []
