"""Hand-off directories for the PnP path (handoff.load_batch_fine, register_dir.py --method): host logic only."""
import os
import subprocess
import sys

import numpy as np

from deepi2p_b200 import handoff, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def write_pnp_dir(path, n_frames=4, n_points=2048):
    """A save_record directory with simulated fine predictions (ragged clouds, both P shapes)."""
    recs = []
    for i in range(n_frames):
        s = synthetic.make_sample(200 + i, n_points=n_points + 37 * i)
        fine = synthetic.make_fine_labels(s, noise=0.3, seed=i)
        name = "%06d_%02d" % (i * 10, i % 2)
        P = s["P_gt"][:3] if i % 2 else s["P_gt"]
        handoff.save_record(str(path), name, s["points"], s["pred"], s["gt"], fine, fine, s["K"], P)
        recs.append((name, s, fine))
    return recs


def test_load_batch_fine_rows(tmp_path):
    recs = write_pnp_dir(tmp_path)
    b = handoff.load_batch_fine(str(tmp_path))
    assert b["names"] == [n for n, _, _ in recs]
    assert b["coarse"].dtype == np.int8 and b["fine"].dtype == np.int32
    for s, (name, smp, fine) in enumerate(recs):
        n = smp["points"].shape[1]
        assert b["n_pts"][s] == n
        # registration_pnp.py:185-189 reads rows 0-2, 3 and 5
        np.testing.assert_array_equal(b["xyz"][s, :, :n], smp["points"])
        np.testing.assert_array_equal(b["coarse"][s, :n], (smp["pred"] == 1).astype(np.int8))
        np.testing.assert_array_equal(b["fine"][s, :n], fine)
        assert (b["coarse"][s, n:] == 0).all() and (b["fine"][s, n:] == 0).all()
        np.testing.assert_array_equal(b["P_gt"][s], smp["P_gt"])


def test_cli_refuses_fine_rows_for_the_frustum_solver(tmp_path):
    """Grid cell indices are not in/out labels: --method lsq with a fine row is an error before any GPU work."""
    write_pnp_dir(tmp_path, n_frames=1, n_points=64)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "register_dir.py"), str(tmp_path), "--H", "160",
                        "--W", "512", "--labels", "fine_prediction"], capture_output=True, text=True)
    assert r.returncode == 2 and "--method pnp" in r.stderr
