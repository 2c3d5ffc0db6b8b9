"""K2's capacity switches and fallback paths against the pixel oracle (oracle/softgl.c).

The render kernel (csrc/raster.cuh) picks between two code paths at several capacity thresholds: candidate lists
per half-tile (MWB_TILE_CAP) or the generic scan, a depth-sorted or draw-order visiting order (MWB_SORT_LIMIT),
triangle records in shared memory or in HBM (tri_cap), staged or L2-read static quads, binned or unbinned mesh lists,
one block per frame or a frame cut into bands, and whole-frame boxes for triangles with a vertex behind the eye.  The
scenes below are built to take one side of a switch with a wide margin, and a census (float64 numpy over the oracle's
draw list, projected with the env's own camera) proves that they do; each quantity is a bound in the direction that
makes the claim safe.  Every scene is rendered on the host build of the kernels, by the drop-in class on the GPU
(N = 1: the frame is cut into several blocks) and by an engine with 12 x SM envs (one block per frame).

Not reached by any scene: a mesh whose half-tile bins would need more than MWB_BIN_REFS x mesh_cap references, where
mesh_cap is the triangle count of the largest mesh prototype in the handle (6 x 208 = 1248 for a level whose only mesh
is a Key, 6 x 1152 = 6912 for the building).  Binning is only tried for more than 64 kept triangles.  For close-ups
of the shipped meshes at 160 x 120 the census's lower bound of references (half-tiles with a pixel centre inside a kept
triangle) stays far below the limit: at most about 190 for a Key and 1700 for the building, over a range of sizes,
distances and headings.  Its upper bound (bounding boxes) does exceed it, so the limit is not proven unreachable.
Not proven either: a flush of the exact-phase queue in the middle of a half-tile (more than MWB_EQ_CAP = 96 undecided
(pixel, triangle) items in one warp).  The crowded scene at 16 samples may reach it, but which pixels stay undecided
depends on the kernel's conservative bounds, which the census does not model.
"""
import math
import re

import numpy as np
import pytest

from miniworld_b200.entity import Agent, Ball, Box, Key
from miniworld_b200.world import MiniWorldEnv

MAX_SLOTS = 65535        # csrc/raster_core.cuh MWB_MAX_SLOTS: slots are 16-bit, id 0xFFFF is the sky
TILE_CAP = 16            # csrc/raster.cuh MWB_TILE_CAP
SORT_LIMIT = 512         # csrc/raster.cuh MWB_SORT_LIMIT
MAX_BINS = 640           # csrc/state.h MWB_MAX_BINS


# ---------------------------------------------------------------------------------------------------- scenes
class _PosedAgent(Agent):
    """An Agent whose camera parameters `cam` override the defaults that reset() gives every agent (it calls
    randomize() on each entity after _gen_world())."""

    def __init__(self, cam):
        super().__init__()
        self.cam = cam

    def randomize(self, params, rng):
        super().randomize(params, rng)
        for k, v in self.cam.items():
            setattr(self, k, v)


class _Scene(MiniWorldEnv):
    """A level whose world is fixed by the test: rooms and entities at given poses, the agent at `pose`
    ((x, z), dir) with the camera parameters `cam` overriding Agent()'s defaults."""

    def __init__(self, pose=((1.0, 15.0), 0.0), cam=None, **kw):
        self.pose, self.cam = pose, dict(cam or {})
        super().__init__(**kw)

    def _place_agent(self):
        (x, z), d = self.pose
        self.agent = _PosedAgent(self.cam)
        self.place_agent(pos=np.array([x, 0.0, z]), dir=d)


class Crowded(_Scene):
    """S1: 15 places along the view axis, each holding two coincident boxes of different colours (equal depth codes:
    the first drawn wins, GL_LESS) that cover the frame's centre half-tiles."""

    def _gen_world(self):
        self.add_rect_room(0, 30, 0, 30)
        for k in range(15):
            for color in ("red", "green"):
                self.place_entity(Box(color, size=[0.6, 2.4, 3.0]), pos=np.array([3.0 + 0.7 * k, 0.0, 15.0]), dir=0.0)
        self._place_agent()


class RoomGrid(_Scene):
    """S2: 9 x 9 rooms of 2.5 m, every neighbour connected by a 1 m portal: more than 250 static quads (triangle
    records in HBM, quads read from L2); more than 512 surviving triangles across the grid's diagonal (draw-order
    visiting), fewer down a row (depth-sorted)."""

    def _gen_world(self):
        n, s = 9, 2.5
        grid = [[self.add_rect_room(c * s, (c + 1) * s, r * s, (r + 1) * s) for c in range(n)] for r in range(n)]
        for r in range(n):
            for c in range(n):
                if c + 1 < n:
                    self.connect_rooms(grid[r][c], grid[r][c + 1], min_z=r * s + 0.7, max_z=r * s + 1.7)
                if r + 1 < n:
                    self.connect_rooms(grid[r][c], grid[r + 1][c], min_x=c * s + 0.7, max_x=c * s + 1.7)
        self._place_agent()


class OneMesh(_Scene):
    """S3: one mesh entity in a room (`ent` = (kind, pos, dir, size))."""

    def __init__(self, ent, **kw):
        self.ent = ent
        super().__init__(**kw)

    def _gen_world(self):
        self.add_rect_room(0, 30, 0, 30)
        kind, pos, d, size = self.ent
        e = Key("yellow") if kind == "key" else Ball("blue", size=size)
        self.place_entity(e, pos=np.array(pos, float), dir=d)
        self._place_agent()


class BallField(_Scene):
    """S4: `n` Balls of 0.9 m on a 1.6 m grid, 8 to 17 m in front of the agent at (1, 0, 15) facing +x."""

    def __init__(self, n, **kw):
        self.n = n
        super().__init__(**kw)

    def _gen_world(self):
        self.add_rect_room(0, 30, 0, 30)
        for k in range(self.n):
            r, c = divmod(k, 6)
            self.place_entity(Ball("red", size=0.9), pos=np.array([9.0 + 1.6 * c, 0.0, 15.0 + 1.6 * (r - 2)]), dir=0.0)
        self._place_agent()


class Corner(_Scene):
    """S5: a 4 x 4 m room with a box and a ball; `carry` = "box" / "ball" puts that object in the agent's hands."""

    def __init__(self, carry=None, **kw):
        self.carry = carry
        super().__init__(**kw)

    def _gen_world(self):
        self.add_rect_room(0, 4, 0, 4)
        self.place_entity(Box("purple", size=0.5), pos=np.array([2.6, 0.0, 1.2]), dir=0.3)
        self.place_entity(Ball("green", size=0.5), pos=np.array([1.3, 0.0, 2.9]), dir=1.1)
        self._place_agent()
        if self.carry is not None:
            ent = Box("yellow", size=0.5) if self.carry == "box" else Ball("red", size=0.5)
            self.max_forward_step = self.params.get_max("forward_step")
            self.place_entity(ent, pos=self._get_carry_pos(self.agent.pos, ent), dir=self.agent.dir)
            self.agent.carrying = ent


# agent poses of S5: touching a wall, wedged in corners facing them, the exact axis / diagonal headings, and the ends of
# the DomainParams camera ranges
R = 0.4                                       # Agent.radius
CORNER_POSES = [
    (((R, 2.0), math.pi), {}),                                  # nose against the x = 0 wall
    (((R, R), 3 * math.pi / 4), {}),                            # wedged in the (0, 0) corner, facing it
    (((4 - R, 4 - R), -math.pi / 4), {}),                       # the (4, 4) corner
    (((2.0, 2.0), 0.0), {}), (((2.0, 2.0), math.pi / 2), {}), (((2.0, 2.0), -math.pi / 2), {}),
    (((2.0, 2.0), math.pi / 4), {}), (((2.0, 2.0), -math.pi / 4), {}),
    (((2.0, 2.0), 0.7), {"cam_pitch": 5.0, "cam_fov_y": 55.0, "cam_fwd_disp": -0.05}),
    (((2.0, 2.0), 2.5), {"cam_pitch": -5.0, "cam_fov_y": 65.0, "cam_fwd_disp": 0.10}),
    (((R, 2.0), math.pi), {"cam_pitch": -5.0, "cam_fov_y": 65.0, "cam_fwd_disp": 0.10}),
]
GRID_POSES = [(((0.6, 1.2), 0.0), {}), (((0.6, 0.6), -math.pi / 4), {}), (((1.2, 0.6), -math.pi / 2), {}),
              (((21.9, 1.2), math.pi), {})]


def scene(name, pose=None, cam=None, device="cuda", **kw):
    """Scene `name` at one agent pose, as a drop-in env (the hostsim_path fixture points it at the host build)."""
    args = dict(device=device, **kw)
    if pose is not None:
        args.update(pose=pose, cam=cam)
    if name == "crowded":
        return Crowded(**args)
    if name == "grid":
        return RoomGrid(**args)
    if name.startswith("balls"):
        return BallField(int(name[5:]), **args)
    if name.startswith("corner"):
        return Corner(carry=name[7:] or None, **args)
    return OneMesh(MESH_CASES[name][0], **args)


# S3: (entity, agent pose, frame size)
MESH_CASES = {
    "key_far": (("key", (12.0, 0.0, 7.2), 0.4, None), ((2.0, 15.0), 0.0), (80, 60)),    # at the frame's edge
    "ball_320": (("ball", (4.0, 0.0, 15.0), 0.0, 2.0), ((1.5, 15.0), 0.0), (320, 240)),
    "ball_160": (("ball", (5.0, 0.0, 15.0), 0.0, 1.2), ((1.0, 15.0), 0.0), (160, 120)),
}


# ---------------------------------------------------------------------------------------------------- census
def project(env, W, H):
    """The frame's draw list (oracle.softgl.draw_list) in float64: image-space (X, Y) (y down), w per vertex, and which
    triangles certainly survive K2's culling and which certainly do not."""
    from oracle import softgl
    pos, _, _, _, _ = softgl.draw_list(env, lambda tex: tex.tex_id)
    P = pos.astype(np.float64)
    a = env.agent
    eye, f = np.asarray(a.cam_pos, np.float64), np.asarray(a.cam_dir, np.float64)
    f = f / np.linalg.norm(f)
    s = np.cross(f, [0.0, 1.0, 0.0])
    s /= np.linalg.norm(s)
    u = np.cross(s, f)
    rel = P - eye
    xe, ye, w = rel @ s, rel @ u, rel @ f
    cot = 1.0 / math.tan(math.radians(a.cam_fov_y) / 2)
    xc, yc = xe * cot * H / W, ye * cot
    with np.errstate(divide="ignore", invalid="ignore"):
        X, Y = (xc / w + 1) * W / 2, (1 - yc / w) * H / 2
    # K2's homogeneous window coordinates (x = X / w, y = Y / w) and clip z (csrc/raster_core.cuh transform_vertex)
    Xh, Yh = (xc + w) * W / 2, (w - yc) * H / 2
    zc = w * (100.0 + 0.04) / (100.0 - 0.04) - 2.0 * 100.0 * 0.04 / (100.0 - 0.04)
    ahead = (w > 0.05).all(1)
    e1, e2 = np.stack([X[:, 1] - X[:, 0], Y[:, 1] - Y[:, 0]], 1), np.stack([X[:, 2] - X[:, 0], Y[:, 2] - Y[:, 0]], 1)
    area = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]          # < 0: counter-clockwise in GL's y-up window = front
    size2 = np.maximum((e1 ** 2).sum(1), (e2 ** 2).sum(1))
    inside = ahead & (np.abs(xc) < 0.999 * w).all(1) & (np.abs(yc) < 0.999 * w).all(1) & (w < 99.0).all(1)
    front = ahead & (area < -1e-4 * size2)                      # robustly front-facing: float32 set-up agrees
    # outside one frustum plane with a margin, or robustly back-facing: certainly culled
    out = ((xc < -1.001 * w).all(1) | (xc > 1.001 * w).all(1) | (yc < -1.001 * w).all(1) | (yc > 1.001 * w).all(1) |
           (ahead & (area > 1e-4 * size2)))
    # kept whatever the vertices' depth (also with vertices behind the eye): strictly inside every frustum plane at some
    # vertex, and a robustly positive set-up determinant (setup_triangle's det, vertices in its (0, 2, 1) order)
    keep_planes = True
    for c in (xc, -xc, yc, -yc, zc, -zc):
        keep_planes = keep_planes & (c < 0.999 * w).any(1)
    v0, v1, v2 = (np.stack([Xh[:, k], Yh[:, k], w[:, k]], 1) for k in (0, 2, 1))
    det = np.einsum("ij,ij->i", v0, np.cross(v1, v2))
    scale = np.abs(v0).sum(1) * np.abs(v1).sum(1) * np.abs(v2).sum(1)
    kept = keep_planes & (det > 1e-6 * scale)
    return dict(X=X, Y=Y, w=w, survive=inside & front, maybe=~out, front=front, ahead=ahead, kept=kept)


def tile_candidates(pr, W, H, sel):
    """Per half-tile (8 x 4), how many of the triangles `sel` that certainly survive contain its centre: the kernel's
    listing test is conservative, so it lists at least these."""
    idx = np.nonzero(sel & pr["survive"])[0]
    X, Y = pr["X"][idx], pr["Y"][idx]
    cx, cy = np.meshgrid(np.arange((W + 7) // 8) * 8 + 4.0, np.arange((H + 3) // 4) * 4 + 2.0)
    cx, cy = cx.reshape(-1, 1), cy.reshape(-1, 1)
    inside = np.ones((cx.shape[0], len(idx)), bool)
    for k in range(3):
        a, b = k, (k + 1) % 3
        # front faces wind clockwise in y-down image space: the interior is on the edges' right
        cross = (X[:, b] - X[:, a]) * (cy - Y[:, a]) - (Y[:, b] - Y[:, a]) * (cx - X[:, a])
        inside &= cross < -1e-6
    return inside.sum(1)


def room_triangles(env):
    """How many triangles of the draw list belong to the rooms (they come first)."""
    from oracle import softgl
    return len(softgl.draw_list(env, lambda tex: tex.tex_id, rooms_only=True)[4])


def mesh_box_halftiles(pr, lo, hi, W, H):
    """Half-tiles covered by the screen box of the surviving triangles lo..hi (a lower bound of the kernel's box), and
    an upper bound of how many triangles it keeps."""
    sel = np.zeros(len(pr["w"]), bool)
    sel[lo:hi] = True
    keep = sel & pr["survive"]
    X, Y = pr["X"][keep], pr["Y"][keep]
    if not keep.any():
        return 0, int((sel & pr["maybe"]).sum()), 0
    x0, x1 = max(0, int(X.min()) + 1), min(W - 1, int(X.max()) - 1)
    y0, y1 = max(0, int(Y.min()) + 1), min(H - 1, int(Y.max()) - 1)
    halves = (x1 // 8 - x0 // 8 + 1) * (y1 // 4 - y0 // 4 + 1) if x1 >= x0 and y1 >= y0 else 0
    return halves, int((sel & pr["maybe"]).sum()), int(keep.sum())


# ---------------------------------------------------------------------------------------------------- runs
def oracle_frame(env, W, H, msaa=8):
    from miniworld_b200.assets import Texture
    from oracle import softgl
    ts = softgl.TextureSet([t.texels for t in Texture.registry])
    try:
        return softgl.render(env, ts, lambda tex: tex.tex_id, W, H, msaa)
    finally:
        ts.close()


def engine_frame(env):
    """RGB and depth of the drop-in env in one render call."""
    eng = env._require_engine()
    env._push_world()
    return eng.render(want_depth=True)


def assert_matches(rgb, depth, want_rgb, want_depth, what):
    d = np.abs(rgb.astype(int) - want_rgb.astype(int))
    assert d.max() <= 1, "%s: %d channel values differ by > 1 LSB (max %d)" % (what, int((d > 1).sum()), int(d.max()))
    assert (d == 0).mean() >= 0.995, "%s: only %.4f of channel values identical" % (what, (d == 0).mean())
    assert np.array_equal(depth, want_depth), "%s: depth differs at %d pixels" % (what, int((depth != want_depth).sum()))
    assert 0 < rgb.mean() < 255


CAMERA = ("cam_height", "cam_fwd_disp", "cam_pitch", "cam_fov_y")      # pack.pack_world(env)["cam"] order


def assert_camera(env, cam):
    """The camera the engine is given is the one the pose asks for."""
    from miniworld_b200 import pack
    pushed = dict(zip(CAMERA, pack.pack_world(env)["cam"]))
    want = dict(cam_height=1.5, cam_fwd_disp=0.0, cam_pitch=0.0, cam_fov_y=60.0)
    want.update(cam or {})
    assert pushed == want, (pushed, want)


def check_scene(name, pose=None, cam=None, W=80, H=60, msaa=8, overflow=False):
    """Render one scene pose through the drop-in class and compare with the oracle; returns (env, frame)."""
    env = scene(name, pose, cam, obs_width=W, obs_height=H, msaa_samples=msaa)
    assert_camera(env, cam)
    rgb, depth = engine_frame(env)
    faults = env._engine.engine.overflow_count()
    if overflow:
        assert faults > 0, "%s: more than %d slots rendered without a capacity fault" % (name, MAX_SLOTS)
    else:
        assert faults == 0, "%s: %d capacity faults" % (name, faults)
        want_rgb, want_depth = oracle_frame(env, W, H, msaa)
        assert_matches(rgb, depth, want_rgb, want_depth, "%s pose %r msaa %d" % (name, pose, msaa))
    return env, (rgb, depth)


# ---------------------------------------------------------------------------------------------------- census tests
def test_census_crowded_half_tiles(softgl_lib):
    env = scene("crowded", device=None)
    pr = project(env, 80, 60)
    best = tile_candidates(pr, 80, 60, np.ones(len(pr["w"]), bool)).max()     # rooms and boxes: all block-resident
    assert best >= 24 > TILE_CAP, best


def test_census_room_grid(softgl_lib):
    env = scene("grid", device=None)
    from miniworld_b200 import pack
    quads = pack.pack_world(env)["quads"]
    assert len(quads) > 250 and quads.nbytes > 16384, (len(quads), quads.nbytes)
    prs = [project(scene("grid", p, c, device=None), 80, 60) for p, c in GRID_POSES]
    # K2 keeps both records of a quad pair if either half survives: an upper bound of its resident records is two per
    # pair (rooms come first in the draw list, every quad as two adjacent triangles) with a half not certainly culled
    records = [2 * int((pr["maybe"][0::2] | pr["maybe"][1::2]).sum()) for pr in prs]
    least = [int(pr["survive"].sum()) for pr in prs]
    assert max(least) > SORT_LIMIT + 100 and min(records) < SORT_LIMIT - 50, (least, records)


def test_census_meshes(softgl_lib):
    for name, (ent, pose, (W, H)) in MESH_CASES.items():
        env = scene(name, pose, device=None)
        pr = project(env, W, H)
        n_room = room_triangles(env)
        halves, most, least = mesh_box_halftiles(pr, n_room, len(pr["w"]), W, H)
        if name == "key_far":
            assert 0 < most <= 64, most                        # unbinned: too few triangles
        elif name == "ball_320":
            assert halves > MAX_BINS + 100 and least > 64, (halves, least)   # unbinned: screen box too large
        else:
            assert halves <= (W // 8) * (H // 4) <= MAX_BINS and least > 64, (halves, least)   # binned


@pytest.mark.parametrize("W,H", [(80, 60), (40, 30)])
def test_census_slot_count(softgl_lib, W, H):
    n26 = project(scene("balls26", device=None), W, H)
    n28 = project(scene("balls28", device=None), W, H)
    # upper bound of the 26-ball frame's slots (every triangle not certainly culled, plus one pad per list) and lower
    # bound of the 28-ball frame's
    assert int(n26["maybe"].sum()) + 27 < MAX_SLOTS < int(n28["survive"].sum()), (n26["maybe"].sum(), n28["survive"].sum())


def test_census_behind_eye(softgl_lib):
    """Triangles that K2 certainly keeps although a vertex lies at or behind the eye plane (whole-frame boxes)."""
    found = []
    for pose, cam in CORNER_POSES:
        env = scene("corner", pose, cam, device=None)
        assert_camera(env, cam)
        pr = project(env, 80, 60)
        found.append(int(((pr["w"] <= 1e-3).any(1) & pr["kept"]).sum()))
    assert sum(found) >= 20 and sum(found[1:3]) >= 4, found     # the wedged-in-a-corner poses among them


# ---------------------------------------------------------------------------------------------------- host build
@pytest.mark.parametrize("msaa", [1, 4, 8, 16])
def test_crowded_half_tiles_host(hostsim_path, softgl_lib, msaa):
    check_scene("crowded", msaa=msaa)


def test_room_grid_host(hostsim_path, softgl_lib):
    for pose, cam in GRID_POSES:
        check_scene("grid", pose, cam)


@pytest.mark.parametrize("name", list(MESH_CASES))
@pytest.mark.parametrize("msaa", [1, 4, 8, 16])
def test_meshes_host(hostsim_path, softgl_lib, name, msaa):
    ent, pose, (W, H) = MESH_CASES[name]
    check_scene(name, pose, W=W, H=H, msaa=msaa)


@pytest.mark.parametrize("n,overflow", [(26, False), (28, True)])
def test_slot_limit_host(hostsim_path, softgl_lib, n, overflow):
    check_scene("balls%d" % n, overflow=overflow)


@pytest.mark.parametrize("name", ["corner", "corner_box", "corner_ball"])
def test_adversarial_cameras_host(hostsim_path, softgl_lib, name):
    for pose, cam in (CORNER_POSES if name == "corner" else CORNER_POSES[3:6]):
        check_scene(name, pose, cam)


# ---------------------------------------------------------------------------------------------------- GPU
def k2_launch_shape(monkeypatch, capfd, make):
    """Build an engine with MWB_DEBUG=1 and read K2's launch shape from mwb_create's report."""
    monkeypatch.setenv("MWB_DEBUG", "1")
    capfd.readouterr()
    obj = make()
    err = capfd.readouterr().err
    monkeypatch.delenv("MWB_DEBUG")
    m = re.findall(r"\[mwb\] K2 (\d+) threads, (\d+)x MSAA: dynamic smem (\d+) B .*parts (\d+)", err)
    assert m, "no K2 report in %r" % err
    threads, msaa, smem, parts = (int(v) for v in m[-1])
    return obj, dict(threads=threads, msaa=msaa, smem=smem, parts=parts)


def big_batch(env, poses_envs, W, H, msaa, N=None):
    """An engine of N (default 12 x SM) envs holding the scene `env` at the given per-env poses (shared static geometry,
    per-env worlds as the drop-in class pushes them)."""
    import torch
    from miniworld_b200 import pack
    from miniworld_b200.engine import MAX_ENTS_CAP, Engine
    N = N or 12 * torch.cuda.get_device_properties(0).multi_processor_count
    worlds = [pack.pack_world(e) for e in poses_envs]
    w0 = worlds[0]
    eng = Engine(N, W, H, msaa, shared_geometry=True, max_rooms=max(8, len(w0["rooms"])),
                 max_quads=max(64, len(w0["quads"])), max_segs=max(64, len(w0["segs"])),
                 max_ents=min(MAX_ENTS_CAP, max(8, len(w0["ents"]))), device=0)
    eng.set_params(env.params)
    eng.sync_assets()
    eng.set_template(w0["rooms"], w0["quads"], w0["segs"])
    eng.set_protos(w0["protos"])
    eng.set_world(np.arange(N), [worlds[k % len(worlds)] for k in range(N)])
    return eng, N


def run_gpu_scene(monkeypatch, capfd, name, poses, W=80, H=60, msaa=8, big=True):
    """(b) every pose through the drop-in class (N = 1, several blocks per frame) against the oracle, then (c) the
    poses spread over 12 x SM envs (one block per frame): a fixed sample of >= 32 envs against the oracle, and every
    sampled env equal to (b)'s frame of its pose."""
    from miniworld_b200 import pack
    envs, single = [], []
    for k, (pose, cam) in enumerate(poses):
        if k == 0:
            (env, frame), shape = k2_launch_shape(monkeypatch, capfd, lambda: check_scene(name, pose, cam, W, H, msaa))
            assert shape["parts"] > 1 and shape["msaa"] == msaa, shape
        else:
            env, frame = check_scene(name, pose, cam, W, H, msaa)
        envs.append(env)
        single.append(frame)
    if big:
        (eng, N), shape = k2_launch_shape(monkeypatch, capfd, lambda: big_batch(envs[0], envs, W, H, msaa))
        assert shape["parts"] == 1, shape
        obs = np.zeros((N, H, W, 3), np.uint8)
        depth = np.zeros((N, H, W, 1), np.float32)
        eng.render(obs=obs, depth=depth)
        assert eng.overflow_count() == 0
        oracle = [oracle_frame(e, W, H, msaa) for e in envs]
        # every pose at spread-out envs, at least 32 envs in all
        per = max(2, -(-32 // len(poses)))
        sample = [k * len(poses) + p for k in np.linspace(0, N // len(poses) - 1, per).astype(int) for p in range(len(poses))]
        cams = eng.get_state()["cam"]
        for i in sample:
            p = i % len(poses)
            assert tuple(cams[i]) == tuple(pack.pack_world(envs[p])["cam"]), (name, i)
            assert_matches(obs[i], depth[i], oracle[p][0], oracle[p][1], "%s env %d of %d" % (name, i, N))
            assert np.array_equal(obs[i], single[p][0]) and np.array_equal(depth[i], single[p][1]), (name, i)
        eng.close()
    for e in envs:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("msaa", [1, 4, 8, 16])
def test_crowded_half_tiles_gpu(libmwb_path, softgl_lib, monkeypatch, capfd, msaa):
    run_gpu_scene(monkeypatch, capfd, "crowded", [(((1.0, 15.0), 0.0), {}), (((1.0, 15.5), 0.0), {})], msaa=msaa)


@pytest.mark.gpu
def test_room_grid_gpu(libmwb_path, softgl_lib, monkeypatch, capfd):
    run_gpu_scene(monkeypatch, capfd, "grid", GRID_POSES)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MESH_CASES))
@pytest.mark.parametrize("msaa", [1, 4, 8, 16])
def test_meshes_gpu(libmwb_path, softgl_lib, monkeypatch, capfd, name, msaa):
    ent, pose, (W, H) = MESH_CASES[name]
    # frames larger than 80 x 60 are always cut into several blocks: the binning cases run at N = 1 only
    if W == 80:
        run_gpu_scene(monkeypatch, capfd, name, [(pose, {})], W, H, msaa)
    else:
        run_gpu_scene(monkeypatch, capfd, name, [(pose, {})], W, H, msaa, big=False)


@pytest.mark.gpu
@pytest.mark.parametrize("n,overflow", [(26, False), (28, True)])
def test_slot_limit_gpu(libmwb_path, softgl_lib, monkeypatch, capfd, n, overflow):
    """The drop-in class (80 x 60, the frame cut into bands), then one block per frame.  At 12 x SM envs the mesh
    triangle lists alone ([N][max_ents][5192] records of 176 B) would take about 40 GB, so the one-block run uses a
    40 x 30 frame, which has fewer than 60 half-tiles and is never cut, at 4 envs."""
    env, _ = check_scene("balls%d" % n, overflow=overflow)
    env.close()
    small = scene("balls%d" % n, device=None, obs_width=40, obs_height=30)
    (eng, N), shape = k2_launch_shape(monkeypatch, capfd, lambda: big_batch(small, [small], 40, 30, 8, N=4))
    assert shape["parts"] == 1, shape
    obs = np.zeros((N, 30, 40, 3), np.uint8)
    depth = np.zeros((N, 30, 40, 1), np.float32)
    eng.render(obs=obs, depth=depth)
    if overflow:
        assert eng.overflow_count() > 0
    else:
        assert eng.overflow_count() == 0
        want_rgb, want_depth = oracle_frame(small, 40, 30)
        for i in range(N):
            assert_matches(obs[i], depth[i], want_rgb, want_depth, "%d balls, 40 x 30, env %d" % (n, i))
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["corner", "corner_box", "corner_ball"])
def test_adversarial_cameras_gpu(libmwb_path, softgl_lib, monkeypatch, capfd, name):
    run_gpu_scene(monkeypatch, capfd, name, CORNER_POSES if name == "corner" else CORNER_POSES[3:6])


@pytest.mark.gpu
def test_maze_large_batch_matches_oracle(libmwb_path, softgl_lib, monkeypatch, capfd):
    """MazeS8 with device resets at 12 x SM envs: HBM triangle lists rendered one block per frame, 32 sampled envs
    against the oracle on host worlds of the same seeds."""
    import torch
    from conftest import golden
    from helpers import make_env
    from miniworld_b200.assets import Texture
    from miniworld_b200.envs import LEVELS
    N = 12 * torch.cuda.get_device_properties(0).multi_processor_count
    env, shape = k2_launch_shape(monkeypatch, capfd, lambda: make_env("maze_dr", golden("maze_dr"), libmwb_path, n=N,
                                                                      want_depth=True))
    assert shape["parts"] == 1 and env.device_reset, shape
    obs = env.render().cpu().numpy()
    depth = env.render_depth().cpu().numpy()
    ts = softgl_lib.TextureSet([t.texels for t in Texture.registry])
    for i in np.linspace(0, N - 1, 32).astype(int):
        m = LEVELS["MiniWorld-MazeS8-v0"](device=None, domain_rand=True)
        m.reset(seed=1000 + int(i))
        rgb, d = softgl_lib.render(m, ts, lambda tex: tex.tex_id)
        assert_matches(obs[i], depth[i], rgb, d, "MazeS8 env %d" % i)
    assert env.engine.overflow_count() == 0
    ts.close()
    env.close()
