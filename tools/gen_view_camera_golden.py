#!/usr/bin/env python
"""Record what the UNMODIFIED reference returns for designed cameras with their own camera attributes, frame size and
sample count, for tests/test_view_cameras.py.

The reference runs through oracle/ref_stub.py under the recording GL (oracle/gl_record.py), as
tools/gen_view_golden.py does.  Along a seeded rollout of each level (actions 0-2 drawn from default_rng(seed), no
episode end), at two steps the script takes each stored 7-column row (x, z, dir, cam_height, cam_fwd_disp, cam_pitch,
cam_fov_y; NaN = leave that attribute as the episode has it), sets `agent.pos = (x, agent.pos[1], z)`,
`agent.dir = dir` and the given camera attributes, calls render_obs(fb) and render_depth(fb) on the reference's own
FrameBuffer(W, H, S) and get_visible_ents() (which renders into obs_fb, the 80 x 60 observation buffer), and puts
everything back before the rollout goes on.  Rows: a raised chase camera behind the agent pitched down 30-70 degrees,
fields of view of 30 and 120, a negative cam_fwd_disp, a camera near the floor below the agent's marker pitched up
60 degrees, a steep -80 degree pitch, and an all-NaN row.  Row j of checkpoint c is rendered at SIZES[(j + c) % 4].
Stored per level in tests/golden/views_cam_<name>.npz: the seed, the actions, the steps, the rows, each frame's size
and samples, the frames (rgb_<k>, depth_<k>) and the visibility masks (bit k = index k of the reference's entity list).

    MWB_REFERENCE_ROOT=<reference checkout> python tools/gen_view_camera_golden.py
"""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_stub  # noqa: E402

# name -> (level id, domain randomisation, seed)
CASES = {"oneroom": ("MiniWorld-OneRoom-v0", False, 31), "fourrooms_dr": ("MiniWorld-FourRooms-v0", True, 32),
         "pickup": ("MiniWorld-PickupObjects-v0", False, 33), "sidewalk": ("MiniWorld-Sidewalk-v0", False, 34),
         "mazes3": ("MiniWorld-MazeS3-v0", False, 35)}
SIZES = [(80, 60, 8), (160, 120, 16), (64, 64, 4), (96, 72, 1)]
STEPS = 8
AT = (3, 7)            # rows are rendered after these many steps
CAM_ATTRS = ("cam_height", "cam_fwd_disp", "cam_pitch", "cam_fov_y")
NAN = math.nan


def rows_for(env, rs):
    """The seven designed rows of one checkpoint."""
    a = env.agent
    rooms = env.rooms

    def inside():
        r = rooms[rs.integers(len(rooms))]
        mx, mz = min(0.3, (r.max_x - r.min_x) / 4), min(0.3, (r.max_z - r.min_z) / 4)
        return rs.uniform(r.min_x + mx, r.max_x - mx), rs.uniform(r.min_z + mz, r.max_z - mz)

    back = rs.uniform(2.0, 3.0)
    chase = (a.pos[0] - back * math.cos(a.dir), a.pos[2] + back * math.sin(a.dir), a.dir,
             rs.uniform(2.5, 4.0), 0.0, -rs.uniform(30, 70), NAN)
    return np.array([
        chase,
        inside() + (rs.uniform(-4, 4), NAN, NAN, NAN, 30.0),
        inside() + (rs.uniform(-4, 4), NAN, NAN, rs.uniform(-10, 10), 120.0),
        inside() + (rs.uniform(-4, 4), NAN, -rs.uniform(0.3, 1.0), NAN, NAN),
        inside() + (rs.uniform(-4, 4), 0.05, NAN, 60.0, NAN),
        inside() + (rs.uniform(-4, 4), 3.0, NAN, -80.0, 90.0),
        inside() + (rs.uniform(-4, 4), NAN, NAN, NAN, NAN),
    ], np.float64)


def record(name):
    level, dr, seed = CASES[name]
    env = ref_stub.make_reference_env(level, record=True, domain_rand=dr)
    from miniworld.opengl import FrameBuffer        # importable once the stub has put the reference on sys.path
    env.reset(seed=seed)
    rs = np.random.default_rng(seed)
    actions = rs.integers(0, 3, STEPS).astype(np.int32)
    rows, size, vis, frames = [], [], [], {}
    fbs = {}
    for t in range(STEPS):
        _, _, term, trunc, _ = env.step(int(actions[t]))
        assert not (term or trunc), "episode ended: pick another seed"
        if t + 1 not in AT:
            continue
        c = AT.index(t + 1)
        for j, row in enumerate(rows_for(env, rs)):
            W, H, S = SIZES[(j + c) % len(SIZES)]
            if (W, H, S) not in fbs:
                fbs[(W, H, S)] = FrameBuffer(W, H, S)
            fb = fbs[(W, H, S)]
            agent = env.agent
            saved = (np.array(agent.pos), agent.dir) + tuple(getattr(agent, k) for k in CAM_ATTRS)
            agent.pos = np.array([row[0], saved[0][1], row[1]])
            agent.dir = float(row[2])
            for k, v in zip(CAM_ATTRS, row[3:]):
                if not math.isnan(v):
                    setattr(agent, k, float(v))
            k = len(rows)
            frames["rgb_%d" % k] = np.array(env.render_obs(fb), np.uint8)
            frames["depth_%d" % k] = np.array(env.render_depth(fb), np.float32)
            vis.append(sum(1 << env.entities.index(e) for e in env.get_visible_ents()))
            agent.pos, agent.dir = saved[0], saved[1]
            for key, v in zip(CAM_ATTRS, saved[2:]):
                setattr(agent, key, v)
            rows.append(row)
            size.append((W, H, S))
    out = os.path.join(ROOT, "tests", "golden", "views_cam_%s.npz" % name)
    np.savez_compressed(out, level=np.array(level), domain_rand=np.array(dr), seed=np.array(seed), actions=actions,
                        at=np.array(AT, np.int32), rows=np.array(rows), size=np.array(size, np.int32),
                        vis=np.array(vis, np.int64), **frames)
    print("wrote %s (%d bytes)" % (out, os.path.getsize(out)))


def main():
    if not ref_stub.reference_available():
        sys.exit("reference checkout not found (set MWB_REFERENCE_ROOT)")
    for name in sys.argv[1:] or CASES:
        record(name)


if __name__ == "__main__":
    main()
