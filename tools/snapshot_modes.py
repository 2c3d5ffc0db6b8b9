"""Snapshot blobs of every run-time mode combination, on the host build of the kernels (CPU only).

For each batch (single OneRoom, FourRooms, PickupObjects and MazeS3; a static and a dynamic two-level table; MazeS2 +
OneRoom with per-env worlds) and each combination of episode seeds, maze layouts, start poses, reset draws, goal
distance and the state bank that its levels allow, this seeds a 4-env batch, writes pending entries for every mode that
is on, resets three envs so that they take them, writes a second set, steps 20 times and takes a snapshot.  The blobs
go to one .npz keyed by batch and modes, so that two revisions can be compared byte for byte:

    python tools/snapshot_modes.py OUT.npz           # in each tree
    python tools/snapshot_modes.py --compare A.npz B.npz

Blobs of Maze levels differ between two runs of the same revision unless both run with MALLOC_PERTURB_=85 in their
environment.  Even then, those of the MazeS2 + OneRoom batch with per-env worlds differ in a few hundred bytes between
two runs of one revision, so compare those keys against such a pair."""
import argparse
import itertools
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCHES = {
    "oneroom": ("MiniWorld-OneRoom-v0", {}),
    "fourrooms": ("MiniWorld-FourRooms-v0", {}),
    "pickup": ("MiniWorld-PickupObjects-v0", {}),
    "mazes3": ("MiniWorld-MazeS3-v0", {}),
    "table_static": (["MiniWorld-OneRoom-v0", "MiniWorld-PickupObjects-v0"], {}),
    "table_dynamic": (["MiniWorld-OneRoom-v0", "MiniWorld-PickupObjects-v0"], dict(dynamic_levels=True)),
    "worlds": (["MiniWorld-MazeS2-v0", "MiniWorld-OneRoom-v0"], dict(per_env_worlds=True)),
}
MODES = ("episode_seeds", "maze_layouts", "start_poses", "reset_draws", "goal_distance", "state_bank")


def _pending(env, k):
    ids = [0, 1, 2]
    if env.dynamic_levels:
        env.set_level_weights([1.0, 2.0])
        env.set_env_level([0], 1)
    if env.episode_seeds:
        env.set_env_seed([1, 2], [17 + k, 23 + k])
    if env.maze_layouts:
        rows, cols = env.maze_shape
        env.set_env_maze([0, 2], np.full((rows, cols), 1 + k, np.uint8), goal_cell=cols - 1, agent_cell=0)
    if env.start_poses:
        env.set_env_pose([1], "agent", 1.5 + k, 1.25, 0.5)
    if env.reset_draws:
        env.set_env_draws([0, 2], 0, float(k))
    if env.state_bank:
        env.save_states([3], [k])
        env.set_env_state([2], k)
    return ids


def run(out):
    lib = subprocess.check_output([os.path.join(ROOT, "tests", "hostsim", "build.sh")]).decode().strip().splitlines()[-1]
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    from miniworld_b200.engine import RNG_DTYPE, rng_state_of
    engine._override_library_for_tests(lib)
    blobs = {}
    for name, (level, kw) in BATCHES.items():
        for on in itertools.product((False, True), repeat=len(MODES)):
            modes = {m: (2 if m == "state_bank" else True) for m, o in zip(MODES, on) if o}
            try:
                env = BatchedMiniWorld(level, 4, **kw, **modes)
            except ValueError:                      # a mode the batch's levels do not allow
                continue
            rng = np.random.default_rng(7)
            env.engine.seed(np.arange(4), np.array([rng_state_of(100 + i) for i in range(4)], RNG_DTYPE))
            env.engine.reset()
            env._seeded = True
            env.engine.reset(_pending(env, 0))
            _pending(env, 1)
            for _ in range(20):
                env.step_host(rng.integers(0, env.action_space.n, 4).astype(np.int32), render=False)
            key = "%s:%s" % (name, "+".join(modes) or "none")
            blobs[key] = env.snapshot()
            env.close()
            print(key, blobs[key].size, flush=True)
    np.savez_compressed(out, **blobs)


def compare(a, b):
    with np.load(a) as x, np.load(b) as y:
        if sorted(x.files) != sorted(y.files):
            print("different keys:", sorted(set(x.files) ^ set(y.files)))
            return 1
        bad = 0
        for k in x.files:
            p, q = x[k], y[k]
            if p.shape != q.shape:
                print("%s: %d bytes against %d" % (k, p.size, q.size))
                bad += 1
            elif not np.array_equal(p, q):
                print("%s: %d of %d bytes differ" % (k, int((p != q).sum()), p.size))
                bad += 1
        print("%d blobs, %d differ" % (len(x.files), bad))
        return 1 if bad else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("out", nargs="?")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    sys.exit(compare(*args.compare) if args.compare else run(args.out))
