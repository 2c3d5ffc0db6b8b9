#!/usr/bin/env python
"""Record what the UNMODIFIED reference returns for designed camera poses, for tests/test_views.py.

The reference runs through oracle/ref_stub.py under the recording GL (oracle/gl_record.py), as
oracle/gen_reference_golden.py does.  Along a seeded rollout of each level (actions 0-2 drawn from default_rng(seed),
no episode end), at two steps the script moves the agent to each stored row -- `agent.pos = (x, agent.pos[1], z)`,
`agent.dir = dir` -- calls render_obs(), render_depth() and get_visible_ents(), and puts the pose back before the
rollout goes on.  Rows: a point inside a room, one against a wall facing it, one 1.2 m from a non-agent entity facing
it (the meshes of PickupObjects) and one outside the floor plan.  Stored per level in tests/golden/views_<name>.npz:
the seed, the actions, the steps, the rows, the frames, the depth maps and the visibility masks (bit k = index k of
the reference's entity list).

    MWB_REFERENCE_ROOT=<reference checkout> python tools/gen_view_golden.py
"""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_stub  # noqa: E402

# name -> (level id, domain randomisation, seed)
CASES = {"oneroom": ("MiniWorld-OneRoom-v0", False, 21), "fourrooms_dr": ("MiniWorld-FourRooms-v0", True, 22),
         "pickup": ("MiniWorld-PickupObjects-v0", False, 23), "sidewalk": ("MiniWorld-Sidewalk-v0", False, 24),
         "mazes3": ("MiniWorld-MazeS3-v0", False, 25)}
STEPS = 8
AT = (2, 6)            # rows are rendered after these many steps


def rows_for(env, rs):
    """The four designed rows of one checkpoint."""
    agent = env.agent
    rooms = env.rooms
    r = rooms[rs.integers(len(rooms))]
    mx, mz = min(0.3, (r.max_x - r.min_x) / 4), min(0.3, (r.max_z - r.min_z) / 4)
    inside = (rs.uniform(r.min_x + mx, r.max_x - mx), rs.uniform(r.min_z + mz, r.max_z - mz), rs.uniform(-4, 4))
    w = rooms[rs.integers(len(rooms))]
    wall = (float(w.min_x) + 0.02, rs.uniform(w.min_z + mz, w.max_z - mz), math.pi)        # at its -x wall, facing it
    others = [e for e in env.entities if e is not agent]
    e = others[rs.integers(len(others))]
    a = rs.uniform(0, 2 * math.pi)
    eye = np.array([e.pos[0] + 1.2 * math.cos(a), e.pos[2] + 1.2 * math.sin(a)])
    d = np.array([e.pos[0], e.pos[2]]) - eye
    facing = (eye[0], eye[1], math.atan2(-d[1], d[0]))
    hi_x = max(float(q.max_x) for q in rooms)
    mid_z = float(np.mean([q.mid_z for q in rooms]))
    outside = (hi_x + 4.0, mid_z, rs.uniform(-4, 4))
    return np.array([inside, wall, facing, outside], np.float64)


def record(name):
    level, dr, seed = CASES[name]
    env = ref_stub.make_reference_env(level, record=True, domain_rand=dr)
    env.reset(seed=seed)
    rs = np.random.default_rng(seed)
    actions = rs.integers(0, 3, STEPS).astype(np.int32)
    rows, rgb, depth, vis = [], [], [], []
    for t in range(STEPS):
        _, _, term, trunc, _ = env.step(int(actions[t]))
        assert not (term or trunc), "episode ended: pick another seed"
        if t + 1 not in AT:
            continue
        for row in rows_for(env, rs):
            agent = env.agent
            pos, dir_ = np.array(agent.pos), agent.dir
            agent.pos = np.array([row[0], pos[1], row[1]])
            agent.dir = float(row[2])
            rgb.append(np.array(env.render_obs()))
            depth.append(np.array(env.render_depth(), np.float32))
            vis.append(sum(1 << env.entities.index(e) for e in env.get_visible_ents()))
            agent.pos, agent.dir = pos, dir_
            rows.append(row)
    out = os.path.join(ROOT, "tests", "golden", "views_%s.npz" % name)
    np.savez_compressed(out, level=np.array(level), domain_rand=np.array(dr), seed=np.array(seed), actions=actions,
                        at=np.array(AT, np.int32), rows=np.array(rows), rgb=np.array(rgb, np.uint8),
                        depth=np.array(depth, np.float32), vis=np.array(vis, np.int64))
    print("wrote %s (%d bytes)" % (out, os.path.getsize(out)))


def main():
    if not ref_stub.reference_available():
        sys.exit("reference checkout not found (set MWB_REFERENCE_ROOT)")
    for name in CASES:
        record(name)


if __name__ == "__main__":
    main()
