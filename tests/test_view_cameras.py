"""Designed cameras with their own camera attributes, frame size and sample count (mwb_render_views_at /
mwb_visible_ents_from_at, BatchedMiniWorld.render_views(size=, samples=) with 7-column rows, MiniWorldEnv.render_view
with camera attributes): NaN columns give the 3-column bytes, the unmodified reference's frames at other sizes and
sample counts, the pixel oracle, the skip rule at its boundaries, no state change and the argument checks.  CPU cases
run the kernels' host build; `gpu` cases run libmwb.so on the device."""
import copy
import math
import os

import numpy as np
import pytest

from level_parity import seed_reset
from test_views import LEVEL_IDS, agent_rows, floor_rows, make, room_point

NAN = math.nan


def seven(rows, intr=(NAN, NAN, NAN, NAN)):
    """[.., 3] rows -> [.., 7] rows with the given intrinsic columns (broadcast)."""
    rows = np.asarray(rows, np.float64)
    tail = np.broadcast_to(np.asarray(intr, np.float64), rows.shape[:-1] + (4,))
    return np.ascontiguousarray(np.concatenate([rows, tail], -1))


# ---------------------------------------------------------------------------------------------------- CPU: NaN columns
@pytest.mark.parametrize("level,dr", [(lv, dr) for lv in LEVEL_IDS for dr in (False, True)
                                      if not (dr and lv == "MiniWorld-Sign-v0")])     # Sign has no randomisation
def test_nan_and_episode_columns_give_the_three_column_bytes(hostsim_path, level, dr):
    """All-NaN 7-column rows, and rows that repeat the episode's own camera values, render, depth and query exactly what
    the 3-column rows do."""
    env = make(level, 3, domain_rand=dr)
    rows = np.stack([agent_rows(env), floor_rows(env, np.random.default_rng(1))])
    want, wd = env.render_views(rows, depth=True)
    cam = env.get_state()["cam"]                     # (cam_height, cam_fwd_disp, cam_pitch, cam_fov_y) per env
    for r7 in (seven(rows), np.ascontiguousarray(np.concatenate([rows, np.broadcast_to(cam, (2,) + cam.shape)], -1))):
        got, gd = env.render_views(r7, depth=True)
        assert np.array_equal(got, want) and np.array_equal(gd, wd), level
        m = np.zeros(3, np.uint32)
        assert np.array_equal(env.visible_ents(out=m, poses=r7[1]),
                              env.visible_ents(out=np.zeros(3, np.uint32), poses=rows[1]))
    env.close()


# ---------------------------------------------------------------------------------------------------- CPU: reference goldens
GOLDEN_CAMS = ["oneroom", "fourrooms_dr", "pickup", "sidewalk", "mazes3"]


@pytest.mark.parametrize("name", GOLDEN_CAMS)
def test_reference_camera_goldens(hostsim_path, name):
    """tests/golden/views_cam_*.npz (tools/gen_view_camera_golden.py): what the unmodified reference's
    render_obs(FrameBuffer(W, H, S)) / render_depth(...) / get_visible_ents() returned with the agent moved to 7-column
    rows -- chase cameras pitched down 30-70 degrees, FOV 30 and 120, negative cam_fwd_disp, a floor camera pitched up
    60, a -80 pitch and NaN columns -- at 80x60/8, 160x120/16, 64x64/4 and 96x72/1.  Frames within 1 LSB and mostly
    identical, depth and visibility identical."""
    from conftest import GOLDEN
    with np.load(os.path.join(GOLDEN, "views_cam_%s.npz" % name)) as z:
        g = {k: z[k] for k in z.files}
    env = make(str(g["level"]), 1, seed=int(g["seed"]), steps=0, domain_rand=bool(g["domain_rand"]))
    per = len(g["rows"]) // len(g["at"])
    k = 0
    for t, a in enumerate(g["actions"]):
        env.step_host(np.array([a], np.int32), render=False)
        if t + 1 not in g["at"]:
            continue
        for _ in range(per):
            W, H, S = (int(v) for v in g["size"][k])
            row = np.ascontiguousarray(g["rows"][k][None])
            got, gd = env.render_views(row, depth=True, size=(W, H), samples=S)
            d = np.abs(got[0].astype(int) - g["rgb_%d" % k].astype(int))
            assert got.shape == (1, H, W, 3)
            assert d.max() <= 1 and (d == 0).mean() > 0.99, (name, k, d.max(), (d == 0).mean())
            assert np.array_equal(gd[0], g["depth_%d" % k]), (name, k)
            mask = env.visible_ents(out=np.zeros(1, np.uint32), poses=row)
            assert int(mask[0]) == int(g["vis"][k]), (name, k)
            k += 1
    assert k == len(g["rows"])
    env.close()


# ---------------------------------------------------------------------------------------------------- CPU: pixel oracle
def oracle_view(softgl, env, ts, row, W, H, S, render_agent=False):
    """softgl's render of `env` with a copy of the agent moved to the 7-column row; the marker at the real pose."""
    lst = softgl.draw_list(env, lambda tex: tex.tex_id, agent_marker=render_agent)
    moved = copy.copy(env)
    moved.agent = copy.copy(env.agent)
    moved.agent.pos = np.array([row[0], env.agent.pos[1], row[1]])
    moved.agent.dir = row[2]
    for name, v in zip(("cam_height", "cam_fwd_disp", "cam_pitch", "cam_fov_y"), row[3:]):
        if not math.isnan(v):
            setattr(moved.agent, name, float(v))
    return softgl._run(moved, ts, lst, W, H, S)


ORACLE_SIZES = [(80, 60, 8), (160, 120, 16), (64, 64, 4), (96, 72, 1), (200, 150, 8), (240, 180, 4)]


@pytest.mark.parametrize("level", ["MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0", "MiniWorld-Sidewalk-v0"])
def test_random_cameras_match_the_oracle(hostsim_path, softgl_lib, level):
    """Random rows, camera attributes, sizes (up to 240x180, beyond the 160x120 mesh binning is sized for) and sample
    counts: the drop-in render_view vs the pixel oracle (<= 1 LSB, depth identical), and the batched render_views of the
    same episode equals the drop-in byte for byte."""
    from miniworld_b200.assets import Texture
    from miniworld_b200.envs import LEVELS
    env = LEVELS[level]()
    env.reset(seed=12)
    batch = make(level, 1, seed=12, steps=0)
    for a in [2, 2, 1, 2, 0, 2]:
        env.step(a)
        batch.step_host(np.array([a], np.int32), render=False)
    ts = softgl_lib.TextureSet([t.texels for t in Texture.registry])
    rs = np.random.default_rng(5)
    for k, (W, H, S) in enumerate(ORACLE_SIZES):
        r = env.rooms[rs.integers(len(env.rooms))]
        intr = [rs.uniform(0.2, 3.0), rs.uniform(-1.0, 0.6), rs.uniform(-75, 75), rs.uniform(20, 130)]
        for j in rs.choice(4, rs.integers(0, 3), replace=False):
            intr[j] = NAN
        row = room_point(r, rs) + (rs.uniform(-4, 4),) + tuple(intr)
        ra = bool(k & 1)
        kw = {n: (None if math.isnan(v) else v) for n, v in zip(("cam_height", "cam_fwd_disp", "cam_pitch", "cam_fov_y"),
                                                                 intr)}
        rgb, depth = env.render_view(*row[:3], render_agent=ra, size=(W, H), samples=S, **kw)
        want, wd = oracle_view(softgl_lib, env, ts, row, W, H, S, ra)
        assert rgb.shape == (H, W, 3)
        assert np.abs(rgb.astype(int) - want.astype(int)).max() <= 1, (k, row)
        assert np.array_equal(depth, wd), (k, row)
        got, gd = batch.render_views(np.array([row]), render_agent=ra, depth=True, size=(W, H), samples=S)
        assert np.array_equal(got[0], rgb) and np.array_equal(gd[0], depth), k
    ts.close()
    env.close()
    batch.close()


def test_other_formats_and_a_second_size(hostsim_path):
    """cwh and grey batches at another size: the frames are render()'s conversion of the hwc frames of that size, and a
    call at the batch's own size after a larger one still equals render() (the staging only grows)."""
    rs = np.random.default_rng(0)
    ref = make("MiniWorld-PickupObjects-v0", 3, domain_rand=True)
    rows = seven(floor_rows(ref, rs), (2.0, NAN, -20.0, 90.0))
    hwc = ref.render_views(rows, size=(120, 90), samples=4)
    for fmt in ("cwh", "grey"):
        env = make("MiniWorld-PickupObjects-v0", 3, domain_rand=True, obs_format=fmt)
        got = env.render_views(rows, size=(120, 90), samples=4)
        if fmt == "cwh":
            assert got.shape == (3, 3, 120, 90) and np.array_equal(got, hwc.transpose(0, 3, 2, 1))
        else:
            assert got.shape == (3, 90, 120, 1) and got.dtype == np.float64
        env.close()
    own = np.zeros(ref.obs_shape, ref.obs_dtype)
    ref.engine.render(obs=own)
    assert np.array_equal(ref.render_views(agent_rows(ref)), own)
    ref.close()


# ---------------------------------------------------------------------------------------------------- CPU: env params
def test_nan_columns_follow_each_envs_merged_params(hostsim_path):
    """With per-env domain-randomisation params, NaN columns take each env's own merged camera params: the all-NaN row
    equals the 3-column row and equals the row that spells those values out."""
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld("MiniWorld-FourRooms-v0", 4, env_params=True)
    env.set_env_param(np.arange(4), "cam_height", default=[1.0, 1.5, 2.0, 2.5])
    env.set_env_param(np.arange(4), "cam_fov_y", default=[40.0, 60.0, 80.0, 100.0])
    seed_reset(env, [3, 4, 5, 6])
    cam = env.get_state()["cam"]
    assert np.array_equal(cam[:, 0], [1.0, 1.5, 2.0, 2.5]) and np.array_equal(cam[:, 3], [40, 60, 80, 100])
    rows = floor_rows(env, np.random.default_rng(2))
    want, wd = env.render_views(rows, depth=True, size=(96, 72), samples=4)
    for r7 in (seven(rows), np.ascontiguousarray(np.concatenate([rows, cam], 1))):
        got, gd = env.render_views(r7, depth=True, size=(96, 72), samples=4)
        assert np.array_equal(got, want) and np.array_equal(gd, wd)
    other = env.render_views(seven(rows, (NAN, NAN, NAN, 60.0)), size=(96, 72), samples=4)
    assert np.array_equal(other[1], want[1]) and not np.array_equal(other[0], want[0])
    env.close()


# ---------------------------------------------------------------------------------------------------- CPU: skipped rows
def test_skip_rule_boundaries(hostsim_path):
    """fov 0 and 180, pitch +-90, +-inf in any intrinsic column and NaN in x / z / dir skip the row (frame, depth and
    mask untouched); fov just inside (0, 180), pitch just inside +-90 and NaN intrinsics render."""
    env = make("MiniWorld-FourRooms-v0", 2)
    base = agent_rows(env)
    big = np.finfo(np.float64).max
    skipped = [(3, math.inf), (3, -math.inf), (4, math.inf), (4, -math.inf), (5, 90.0), (5, -90.0), (5, 1e300),
               (5, math.inf), (6, 0.0), (6, 180.0), (6, -1.0), (6, -math.inf), (6, math.inf), (0, NAN), (1, NAN),
               (2, NAN), (2, math.inf)]
    rendered = [(3, big), (5, 89.999), (5, -89.999), (6, 1e-3), (6, 179.9), (3, NAN), (4, NAN), (5, NAN), (6, NAN)]
    for col, v in skipped + rendered:
        rows = seven(base)
        rows[1, col] = v
        out = np.full((2, 60, 80, 3), 33, np.uint8)
        depth = np.full((2, 60, 80, 1), -1.0, np.float32)
        env.render_views(rows, out=out, depth=depth)
        mask = np.full(2, 7, np.uint32)
        env.visible_ents(out=mask, poses=rows)
        if (col, v) in skipped:
            assert (out[1] == 33).all() and (depth[1] == -1.0).all() and mask[1] == 7, (col, v)
        else:
            assert not (depth[1] == -1.0).all(), (col, v)
        assert not (out[0] == 33).all() and mask[0] != 7
    env.close()
    from miniworld_b200.envs import LEVELS
    single = LEVELS["MiniWorld-OneRoom-v0"]()
    single.reset(seed=1)
    for kw in (dict(cam_fov_y=0.0), dict(cam_fov_y=180.0), dict(cam_pitch=90.0), dict(cam_pitch=-90.0),
               dict(cam_height=math.inf), dict(cam_fwd_disp=-math.inf)):
        with pytest.raises(ValueError, match="render_view"):
            single.render_view(1.0, 1.0, 0.0, **kw)
    single.close()


# ---------------------------------------------------------------------------------------------------- CPU: no state change
def test_camera_views_change_no_state(hostsim_path):
    """A 200-step rollout with a chase view at 160x120/16 and a two-camera view after every step equals a twin without
    them, and the snapshot is unchanged by a call."""
    a = make("MiniWorld-PickupObjects-v0", 2, steps=0, domain_rand=True, want_depth=True)
    b = make("MiniWorld-PickupObjects-v0", 2, steps=0, domain_rand=True, want_depth=True)
    blob = a.snapshot()
    a.render_views(seven(agent_rows(a), (2.5, -3.0, -25.0, NAN)), render_agent=True, size=(160, 120), samples=16)
    assert np.array_equal(a.snapshot(), blob)
    rs = np.random.default_rng(3)
    for t in range(200):
        acts = rs.integers(0, 5, 2).astype(np.int32)
        oa, ob = a.step_host(acts), b.step_host(acts)
        rows = agent_rows(a)
        a.render_views(seven(rows, (2.5, -3.0, -25.0, NAN)), render_agent=True, size=(160, 120), samples=16)
        a.render_views(np.stack([seven(rows, (NAN, NAN, NAN, 110.0)), seven(rows, (NAN, NAN, NAN, 40.0))]))
        for k in ("obs", "depth", "reward", "terminated", "truncated"):
            assert np.array_equal(oa[k], ob[k]), (t, k)
    assert np.array_equal(a.snapshot(), b.snapshot())
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------------- CPU: sharding
def _shard_worker(rank, port, lib, q):
    import torch.distributed as dist
    from miniworld_b200 import engine
    from miniworld_b200.dist import ShardedMiniWorld
    engine._override_library_for_tests(lib)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=2)
    env = ShardedMiniWorld("MiniWorld-FourRooms-v0", 5, dist=dist)
    env.local.engine.seed(np.arange(env.count), np.array([engine.rng_state_of(9 + env.start + k) for k in range(env.count)],
                                                         engine.RNG_DTYPE))
    env.local.engine.reset()
    rows = seven(np.random.default_rng(0).uniform(1, 12, (2, 5, 3)), (2.0, NAN, -30.0, 100.0))
    out = env.render_views(np.ascontiguousarray(rows[:, env.start:env.start + env.count]), size=(64, 64), samples=4)
    q.put((rank, out))
    dist.barrier()
    env.close()
    dist.destroy_process_group()


def test_sharded_camera_views_equal_one_process(hostsim_path):
    import torch.multiprocessing as mp
    from miniworld_b200.batched import BatchedMiniWorld
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33000 + os.getpid() % 2000
    procs = [ctx.Process(target=_shard_worker, args=(r, port, hostsim_path, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
    one = BatchedMiniWorld("MiniWorld-FourRooms-v0", 5)
    seed_reset(one, [9 + i for i in range(5)])
    rows = seven(np.random.default_rng(0).uniform(1, 12, (2, 5, 3)), (2.0, NAN, -30.0, 100.0))
    want = one.render_views(rows, size=(64, 64), samples=4)
    assert want.shape == (2, 5, 64, 64, 3)
    assert np.array_equal(np.concatenate([got[0], got[1]], 1), want)
    one.close()


# ---------------------------------------------------------------------------------------------------- CPU: errors
def test_argument_errors(hostsim_path):
    from miniworld_b200.engine import EngineError
    env = make("MiniWorld-OneRoom-v0", 2, steps=0)
    rows = seven(agent_rows(env))
    for bad in (rows[:, :5], np.zeros((2, 4)), np.zeros((2, 8))):
        with pytest.raises(ValueError, match="shape"):
            env.render_views(np.ascontiguousarray(bad))
        with pytest.raises(ValueError, match="shape"):
            env.visible_ents(out=np.zeros(2, np.uint32), poses=np.ascontiguousarray(bad))
    for size in ((0, 60), (80, -1), (80,), (80.0, 60), "80x60", (True, 60)):
        with pytest.raises(ValueError, match="size"):
            env.render_views(rows, size=size)
    for s in (0, 2, 3, 32, True):
        with pytest.raises(ValueError, match="samples"):
            env.render_views(rows, samples=s)
    with pytest.raises(ValueError, match="out"):
        env.render_views(rows, size=(64, 48), out=np.zeros((2, 60, 80, 3), np.uint8))
    with pytest.raises(ValueError, match="depth"):
        env.render_views(rows, size=(64, 48), depth=np.zeros((2, 60, 80, 1), np.float32))
    eng, lib = env.engine, env.engine.lib
    obs, p = np.zeros((2, 60, 80, 3), np.uint8), rows.ctypes.data
    mask = np.zeros(2, np.uint32).ctypes.data
    for args, msg in (((p, 5, 1, 80, 60, 8), "row_width must be 3 or 7"), ((p, 7, 1, 0, 60, 8), "width and height must be positive"),
                      ((p, 7, 1, 80, -3, 8), "width and height must be positive"), ((p, 7, 1, 80, 60, 2), "samples must be 1, 4, 8 or 16"),
                      ((p, 7, 0, 80, 60, 8), "views must be positive"), ((None, 7, 1, 80, 60, 8), "null argument")):
        with pytest.raises(EngineError, match=msg):
            eng._check(lib.mwb_render_views_at(eng.h, *args, 0, obs.ctypes.data, None, None))
    with pytest.raises(EngineError, match="null argument"):
        eng._check(lib.mwb_render_views_at(eng.h, p, 7, 1, 80, 60, 8, 0, None, None, None))
    with pytest.raises(EngineError, match="row_width must be 3 or 7"):
        eng._check(lib.mwb_visible_ents_from_at(eng.h, p, 4, mask, None))
    with pytest.raises(EngineError, match="null argument"):
        eng._check(lib.mwb_visible_ents_from_at(eng.h, None, 7, mask, None))
    env.close()
    from miniworld_b200.envs import LEVELS
    single = LEVELS["MiniWorld-OneRoom-v0"]()
    single.reset(seed=1)
    for kw in (dict(size=(0, 60)), dict(samples=3)):
        with pytest.raises(ValueError, match="render_view"):
            single.render_view(1.0, 1.0, 0.0, **kw)
    single.close()


# ---------------------------------------------------------------------------------------------------- GPU
def _gpu_batch(level, n, **kw):
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(level, n, **kw)
    env.reset(seed=0)
    g = torch.Generator(device="cuda").manual_seed(1)
    for _ in range(8):
        env.step(torch.randint(0, 3, (n,), device="cuda", generator=g, dtype=torch.int32))
    return env


def _host_lib():
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return subprocess.check_output([os.path.join(root, "tests", "hostsim", "build.sh")]).decode().strip().splitlines()[-1]


def _random_cameras(env, rs):
    rows = floor_rows(env, rs)
    n = len(rows)
    intr = np.stack([rs.uniform(0.2, 3.0, n), rs.uniform(-1.0, 0.6, n), rs.uniform(-75, 75, n), rs.uniform(20, 130, n)], 1)
    intr[rs.random((n, 4)) < 0.25] = NAN
    return np.ascontiguousarray(np.concatenate([rows, intr], 1))


@pytest.mark.gpu
@pytest.mark.parametrize("level", ["MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0"])
def test_gpu_cameras_equal_the_host_build(libmwb_path, level):
    """At 4096 envs, 7-column rows at 160x120/16, 64x64/4 and 320x240/8 (mesh binning falls back beyond 160x120): a
    sample of envs equals the host build run on those envs' state (<= 1 LSB, depth identical)."""
    import torch
    from miniworld_b200 import engine
    from miniworld_b200.batched import BatchedMiniWorld
    N, pick = 4096, np.array([0, 1, 777, 2048, 4095])
    dev = _gpu_batch(level, N, domain_rand=True)
    rows = _random_cameras(dev, np.random.default_rng(9))
    sizes = [(160, 120, 16), (64, 64, 4), (320, 240, 8)]
    want = [dev.render_views(torch.tensor(rows, device="cuda"), render_agent=True, depth=True, size=(W, H), samples=S)
            for W, H, S in sizes]
    want = [(o[pick].cpu().numpy(), d[pick].cpu().numpy()) for o, d in want]
    blob = dev.snapshot()
    dev.close()
    engine._override_library_for_tests(_host_lib())
    try:
        host = BatchedMiniWorld(level, N, domain_rand=True)
        host.restore(blob)
        for (W, H, S), (o, d) in zip(sizes, want):
            sub = np.full_like(rows, NAN)
            sub[pick] = rows[pick]
            ho, hd = host.render_views(sub, render_agent=True, depth=True, size=(W, H), samples=S)
            assert np.abs(ho[pick].astype(int) - o.astype(int)).max() <= 1 and np.array_equal(hd[pick], d), (W, H, S)
        host.close()
    finally:
        engine._override_library_for_tests(None)


@pytest.mark.gpu
def test_gpu_camera_rows_from_a_busy_side_stream(libmwb_path):
    """7-column rows written by a slow torch kernel on a busy side stream, handed over by stream order, are read in
    order: all-NaN intrinsics give render()'s frames."""
    import torch
    env = _gpu_batch("MiniWorld-FourRooms-v0", 2048)
    obs = env.render().clone()
    st = env.get_state()
    rows = torch.tensor(np.concatenate([np.stack([st["agent_pos"][:, 0], st["agent_pos"][:, 2], st["agent_dir"]], 1),
                                        np.full((2048, 4), NAN)], 1), device="cuda")
    side = torch.cuda.Stream()
    poses = torch.full_like(rows, float("inf"))
    with torch.cuda.stream(side):
        x = torch.randn(2048, 2048, device="cuda")
        for _ in range(20):
            x = x @ x / 2048.0                 # keeps the side stream busy
        poses.copy_(rows + 0.0 * x[:2048, :7].double().nan_to_num(0, 0, 0).clamp(0, 0))
    torch.cuda.current_stream().wait_stream(side)
    out = env.render_views(poses)
    torch.cuda.synchronize()
    assert torch.equal(out, obs)
    env.close()


@pytest.mark.gpu
def test_gpu_chase_views_change_no_state(libmwb_path):
    """A device rollout with a 160x120/16 chase view after every step (and a two-camera 80x60 view) equals a twin without
    the views: observations, depth, rewards and flags every step, the snapshot at the end."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    N = 512
    a = BatchedMiniWorld("MiniWorld-PickupObjects-v0", N, domain_rand=True, want_depth=True)
    b = BatchedMiniWorld("MiniWorld-PickupObjects-v0", N, domain_rand=True, want_depth=True)
    a.reset(seed=3)
    b.reset(seed=3)
    g = torch.Generator(device="cuda").manual_seed(0)
    chase = torch.zeros((N, 7), dtype=torch.float64, device="cuda")
    chase[:, 3:] = torch.tensor([2.5, -3.0, -25.0, NAN], dtype=torch.float64)
    two = torch.full((2, N, 7), NAN, dtype=torch.float64, device="cuda")
    two[0, :, 6], two[1, :, 6] = 110.0, 40.0
    for t in range(100):
        acts = torch.randint(0, 5, (N,), device="cuda", generator=g, dtype=torch.int32)
        oa, ra, ta, ua, ia = a.step(acts)
        oa, ra, ta, ua, da = oa.clone(), ra.clone(), ta.clone(), ua.clone(), ia["depth"].clone()
        ob, rb, tb, ub, ib = b.step(acts)
        assert torch.equal(oa, ob) and torch.equal(da, ib["depth"]), t
        assert torch.equal(ra, rb) and torch.equal(ta, tb) and torch.equal(ua, ub), t
        st = a.get_state()
        chase[:, :3] = torch.tensor(np.stack([st["agent_pos"][:, 0], st["agent_pos"][:, 2], st["agent_dir"]], 1),
                                    device="cuda")
        a.render_views(chase, render_agent=True, size=(160, 120), samples=16)
        two[:, :, :3] = chase[:, :3]
        a.render_views(two)
    torch.cuda.synchronize()
    assert np.array_equal(a.snapshot(), b.snapshot())
    a.close()
    b.close()


@pytest.mark.gpu
def test_gpu_no_overflow_at_wide_fields_of_view(libmwb_path):
    """mwb_overflow_count() is unchanged by 7-column views from rows inside every level's floor plan at fields of view
    up to 120, pitched -60..60, at 80x60/8 and 160x120/16."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    for level in LEVEL_IDS:
        env = BatchedMiniWorld(level, 256)
        env.reset(seed=1)
        before = env.engine.overflow_count()
        rs = np.random.default_rng(5)
        rows = floor_rows(env, rs)
        for fov in (60.0, 90.0, 120.0):
            r7 = seven(rows, (NAN, NAN, NAN, fov))
            r7[:, 5] = rs.uniform(-60, 60, len(rows))
            t = torch.tensor(r7, device="cuda")
            env.render_views(torch.stack([t, t.flip(0)]), render_agent=True, depth=True)
            env.render_views(t, size=(160, 120), samples=16, depth=True)
            env.visible_ents(poses=t)
            torch.cuda.synchronize()
            assert env.engine.overflow_count() == before, (level, fov)
        env.close()
