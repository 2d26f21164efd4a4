"""Development aid: relative position error between the device and the free-running oracle (same Gauss-Seidel order
injected each step, no state ever copied) every 50 steps -- how long a settling pile stays within 1e-4.
usage: python tools/free_run_drift.py boxes 16 | chains 64"""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import edyn_b200 as E
from oracle import oracle as O
from tests import parity as P
kind, n = sys.argv[1], int(sys.argv[2])
scene = E.scenes.boxes_on_plane(n) if kind == "boxes" else E.scenes.hinge_chains(n, n)
w = E.scenes.build_world(scene, max_manifolds=8 * len(scene["bodies"]["kind"]))
o = P.oracle_for(O, scene, threads=os.cpu_count())
nd = scene["dynamic"]
for s in range(1000):
    w.run_phases(E.world.PH_ALL)
    P.oracle_step(O, o, w)
    if s % 50 == 49:
        g, c = w.download_state(aabb=False), o.state()
        err = np.abs(g["pos"][:nd] - c["pos"][:nd]).max(axis=1)
        scale = np.abs(c["pos"][:nd]).max()
        print(f"step {s + 1:4d}  max rel {err.max() / scale:.3e}  bodies beyond 1e-4: {(err / scale > 1e-4).sum():5d} / {nd}   max |v| {np.abs(c['linvel'][:nd]).max():.3f}", flush=True)
