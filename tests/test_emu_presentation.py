"""k_presentation under the CPU emulation of tests/emu, bit for bit against the restatement of the reference's
update_presentation / snap_presentation in tests/presentation/ora_presentation.hpp (tests/emu/presentation.py): awake, kinematic and presentation-less bodies,
negative, zero and positive dt, snaps between updates.  Both sides use glibc's sinf / cosf here, so nothing is exempt."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_emulated_presentation_kernel_equals_the_oracle(O):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emu", "presentation.py")], capture_output=True, text=True,
                       cwd=ROOT, timeout=1500)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["calls"] == 48 and res["mismatched"] == 0, res
