"""Cost of the batched engine's features, measured on one GPU, one study per feature.

    python tools/bench_study.py STUDY [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3] [--episode-steps 20]
                                      [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20] [--bench-only]
    python tools/bench_study.py STUDY --help        (the study's arms and options)

Part 1 runs the study's arms alternately for `--rounds` rounds, device-resident like bench.py's main arm (actions,
observations, rewards and flags stay in device memory).  Every batch resets with seed 1000 and steps with actions
drawn by numpy's generator seeded 12345; torch ops that write run-time arrays draw from a torch generator seeded 3.
A run warms up for `--warmup` steps, then times `--steps` steps between two CUDA events and prints one JSON line:
env-steps/s, K1 / K2 time per launch (mwb_profile), resets per step and the device memory the batch holds per env
(cudaMemGetInfo around its construction and reset), plus what the study adds.  Studies with truncated levels end
every episode after `--episode-steps` steps and start each env's step count staggered, so that a twentieth of the envs
reset in every step instead of all of them in one.  A summary line per arm gives the median and the spread
(min, max) over the rounds of each time the arm's runs have.

Part 2 (with `--baseline-tree DIR`, a built checkout of another revision): `bench.py --gpus 1` (default config) and
`bench.py --gpus 1 --config 4` (MazeS8 with randomisation) of DIR and of this tree, alternately, `--rounds` times
each, then `--dump-outputs` of both compared file by file for both configs.  `--bench-only` runs part 2 alone.
The first line names the card and its power limit.  Nothing is written to either tree (dumps go to a temporary
directory).
"""
import argparse
import filecmp
import inspect
import json
import math
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FOURROOMS, PICKUP, MAZES3, MAZE8 = ("MiniWorld-FourRooms-v0", "MiniWorld-PickupObjects-v0", "MiniWorld-MazeS3-v0",
                                    "MiniWorld-Maze-v0")
MIX4 = [FOURROOMS, "MiniWorld-Hallway-v0", "MiniWorld-OneRoom-v0", PICKUP]
# what the summary lines summarise, where a run has it
TIMES = ("env_steps_per_s", "k1_ms_per_launch", "k2_ms_per_launch", "views_ms_per_call", "views_ms_per_view",
         "all_skipped_ms_per_call", "first_ms", "later_ms", "k1_us_per_launch")


# ---- shared: the card, the batch, the timed run, the profiler, the summary

def card():
    """Name and power limit of GPU 0 (a read-only nvidia-smi query)."""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception:
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown"}


def short_level(name, steps):
    """The level truncated after `steps` steps: frequent resets."""
    from miniworld_b200.envs import LEVELS as REGISTRY
    base = REGISTRY[name]

    def __init__(self, **kw):
        base.__init__(self, **kw)
        self.max_episode_steps = steps
    return type("Short" + base.__name__, (base,), {"__init__": __init__})


def build(level, n, episode_steps=None, **kw):
    """BatchedMiniWorld(level, n, **kw) reset with seed 1000, and the device bytes it holds (cudaMemGetInfo around
    its construction and reset).  With `episode_steps` the level is truncated after that many steps and env i's
    step count starts at i % episode_steps."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    env = BatchedMiniWorld(short_level(level, episode_steps) if episode_steps else level, n, **kw)
    env.reset(seed=1000)
    torch.cuda.synchronize()
    held = free0 - torch.cuda.mem_get_info()[0]
    if episode_steps:
        dev = torch.device("cuda", env.device)
        stagger = torch.as_tensor(env.engine.state_array("step_count"), device=dev)
        stagger.copy_(torch.arange(n, device=dev, dtype=torch.int32) % episode_steps)
    return env, held


def actions(env, args, high=None):
    """The actions of the warm-up and timed steps, below `high` (default: the size of the action space)."""
    import numpy as np
    import torch
    high = env.single_action_space.n if high is None else high
    return torch.as_tensor(np.random.default_rng(12345).integers(0, high, size=(args.warmup + args.steps, env.num_envs),
                                                                 dtype=np.int32), device=torch.device("cuda", env.device))


def generator(env):
    import torch
    gen = torch.Generator(device=torch.device("cuda", env.device))
    gen.manual_seed(3)
    return gen


def episodes_done(env):
    return int(env.get_state()["episodes_done"][0])


def run(arm, env, held, args, step, profile=True, at_start=None):
    """step(t) for the `--warmup` warm-up steps, then the `--steps` timed ones between two CUDA events, with mwb_profile
    on when `profile`.  `at_start()` runs after the warm-up, outside the timed window.  Returns the run's record."""
    import torch
    n = env.num_envs
    for t in range(args.warmup):
        step(t)
    torch.cuda.synchronize()
    env.engine.profile(profile)
    env.engine.profile_read()
    if at_start:
        at_start()
    done0 = episodes_done(env)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(args.warmup, args.warmup + args.steps):
        step(t)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    k1, k2, n1, n2 = env.engine.profile_read()
    env.engine.profile(False)
    rec = {"arm": arm, "envs": n, "steps": args.steps, "env_steps_per_s": n * args.steps / (ms * 1e-3),
           "ms_per_step": ms / args.steps}
    if profile:
        rec.update(k1_ms_per_launch=k1 / max(n1, 1), k2_ms_per_launch=k2 / max(n2, 1),
                   k2_launches_per_step=n2 / args.steps)
    rec.update(resets_per_step=(episodes_done(env) - done0) / args.steps, device_bytes_per_env=held / n)
    return rec


def finish(env, rec):
    """Check that no frame overflowed its triangle lists, close the batch and print the record."""
    assert env.engine.overflow_count() == 0
    env.close()
    print(json.dumps(rec), flush=True)
    return rec


def kernel_ms(fn, names):
    """Device time (ms) per name of the kernels whose names contain it, over one call of fn, with launch counts
    (torch.profiler, CUDA activity only)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in names:
            if name in ev.key:
                total = getattr(ev, "device_time_total", None)
                total = ev.cuda_time_total if total is None else total
                ms, count = out.get(name, (0.0, 0))
                out[name] = (ms + total / 1e3, count + ev.count)
    return out


def summary(recs):
    """One line per arm (and levels, build, config, profiler): the median and the spread (min, max) of every time
    in TIMES its runs have."""
    import numpy as np
    ids = ("levels", "build", "config", "profiler")
    groups = {}
    for r in recs:
        groups.setdefault(json.dumps([r["arm"]] + [r.get(k) for k in ids]), []).append(r)
    for rs in groups.values():
        out = {"summary": rs[0]["arm"], "runs": len(rs)}
        out.update({k: rs[0][k] for k in ids if k in rs[0]})
        for key in TIMES:
            if all(key in r for r in rs):
                v = np.array([r[key] for r in rs])
                out[key] = {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}
        print(json.dumps(out), flush=True)


# ---- part 2: bench.py of a baseline tree and of this tree

def run_bench(tree, label, args, config, dump=None):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps),
           "--warmup", str(args.bench_warmup), "--no-cpu"] + (["--config", str(config)] if config else []) + \
          (["--dump-outputs", dump] if dump else [])
    out = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, check=True).stdout
    line = json.loads([s for s in out.splitlines() if s.startswith("{")][-1])
    rec = {"arm": "bench.py", "build": label, "config": config or "default", "env_steps_per_s": line["value"],
           "ms_per_step": line["ms_per_step"], "k1_ms_per_launch": line["roofline"]["k1_avg_ms"],
           "k2_ms_per_launch": line["roofline"]["kernel_avg_ms"]}
    print(json.dumps(rec), flush=True)
    return rec


def compare_trees(args):
    base = os.path.abspath(args.baseline_tree)
    recs = []
    for _ in range(args.rounds):
        for config in (None, 4):
            recs.append(run_bench(base, "baseline", args, config))
            recs.append(run_bench(ROOT, "this tree", args, config))
    summary(recs)
    for config in (None, 4):
        with tempfile.TemporaryDirectory() as tmp:
            a, b = os.path.join(tmp, "baseline"), os.path.join(tmp, "this")
            run_bench(base, "baseline", args, config, dump=a)
            run_bench(ROOT, "this tree", args, config, dump=b)
            names = sorted(os.listdir(a))
            same = names == sorted(os.listdir(b)) and all(
                filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False) for f in names)
            print(json.dumps({"arm": "dump-outputs", "config": config or "default", "files": names,
                              "byte_identical": same}), flush=True)


# ---- the studies

def configs(args):
    """Throughput of every BASELINE.json config at its per-GPU size (device-resident arm only; bench.py is the main
    benchmark), one run per config and round."""
    table = [   # name, level, envs per GPU, kwargs
        ("config1_hallway", "MiniWorld-Hallway-v0", 1, {}),
        ("config2_oneroom", "MiniWorld-OneRoom-v0", 1024, {}),
        ("config3_fourrooms_depth", FOURROOMS, 4096, {"want_depth": True}),
        ("config4_maze_dr_per_gpu", "MiniWorld-MazeS8-v0", 1024, {"domain_rand": True}),
        ("config5_pickup_160x120_per_gpu", PICKUP, 512, {"obs_width": 160, "obs_height": 120}),
    ]

    def one(name, level, n, kw):
        env, held = build(level, n, **kw)
        acts = actions(env, args)
        rec = run(name, env, held, args, lambda t: env.step(acts[t]))
        rec.update(config=name, level=level, kwargs=kw, device_reset=env.device_reset, k1_ms=rec["k1_ms_per_launch"],
                   k2_ms=rec["k2_ms_per_launch"], episodes_done=round(rec["resets_per_step"] * args.steps),
                   tri_overflow_frames=env.engine.overflow_count())
        return finish(env, rec)
    return [one(*row) for _ in range(args.rounds) for row in table]


def mixed(args):
    """Cost of running several levels in one batch.
      * mixed: one handle of `--envs` envs, the levels in contiguous near-equal blocks (BatchedMiniWorld's default);
      * alone: each level on its own handle with the same per-level env count.
    Each run adds K2's launches per step, its triangle capacity and its block shape, dynamic shared memory and resident
    blocks per SM (the `MWB_DEBUG` report of mwb_create).  The last line of each round compares the mixed step time
    with the sum of the levels' step times."""
    def one(arm, levels, n):
        os.environ["MWB_DEBUG"] = "1"
        sys.stderr.flush()
        saved = os.dup(2)
        with tempfile.TemporaryFile(mode="w+") as f:
            os.dup2(f.fileno(), 2)
            try:
                env, held = build(levels, n)
            finally:
                os.dup2(saved, 2)
                os.close(saved)
                del os.environ["MWB_DEBUG"]
            f.seek(0)
            report = [line.strip() for line in f if line.startswith("[mwb] K2")]
        acts = actions(env, args)
        rec = run(arm, env, held, args, lambda t: env.step(acts[t]))
        cfg = env.engine.cfg
        rec.update(levels=levels if isinstance(levels, list) else [levels], tri_cap=2 * (cfg.max_quads + 6 * cfg.max_ents) + 2,
                   k2_report=report[-1] if report else "")
        return finish(env, rec)

    recs = []
    for _ in range(args.rounds):
        mix = one("mixed", list(args.levels), args.envs)
        alone = [one("alone", lv, args.envs // len(args.levels)) for lv in args.levels]
        parts = sum(a["ms_per_step"] for a in alone)
        print(json.dumps({"arm": "summary", "mixed_ms_per_step": mix["ms_per_step"], "sum_of_levels_ms_per_step": parts,
                          "mixed_over_sum": mix["ms_per_step"] / parts}), flush=True)
        recs += [mix] + alone
    return recs


def level_changes(args):
    """Cost of level changes at resets (BatchedMiniWorld(dynamic_levels=True)) on a mix of levels (default 4096 envs
    over FourRooms, Hallway, OneRoom, PickupObjects, contiguous blocks):
      * static:   level changes off;
      * idle:     level changes on, all weights zero (every reset keeps its level);
      * sampling: level changes on, weights replaced on the device every 50 steps by torch ops (no host sync).
    The sampling and idle runs add how many envs changed level in the timed region."""
    import torch
    levels = list(args.levels)

    def one(arm):
        env, held = build(levels, args.envs, dynamic_levels=arm != "static", level_seed=7)
        acts = actions(env, args)
        gen = generator(env)
        start = []

        def step(t):
            if arm == "sampling" and t % 50 == 0:
                env.level_weights.copy_(torch.rand(len(levels), device=acts.device, generator=gen))
            env.step(acts[t])
        rec = run(arm, env, held, args, step,
                  at_start=None if arm == "static" else lambda: start.append(env.level_tensor.clone()))
        rec["levels"] = levels
        if start:
            rec["envs_whose_level_changed"] = int((env.level_tensor != start[0]).sum())
        return finish(env, rec)
    return [one(arm) for _ in range(args.rounds) for arm in ("static", "idle", "sampling")]


def level_dr(args):
    """Cost of per-level domain randomisation (mwb_level.domain_rand): `--envs` FourRooms envs as a table of three rows.
      * off:    three rows, all with domain_rand off;
      * on:     three rows, all with domain_rand on;
      * ladder: off / on with ranges narrowed to a quarter / on, envs starting on row 0 and moved by weights that torch
                ops rewrite on the device every 50 steps (level changes on, no host sync).
    The ladder runs add how many envs each row holds at the end."""
    import numpy as np
    import torch
    from miniworld_b200.params import DEFAULT_PARAMS
    def rows(arm):
        if arm != "ladder":
            return [{"domain_rand": arm == "on"}] * 3
        narrowed = DEFAULT_PARAMS.copy()          # every range shrunk to a quarter of its width around the default
        for name, q in DEFAULT_PARAMS.params.items():
            if isinstance(q.default, np.ndarray):
                lo, hi = q.default - 0.25 * (q.default - q.min), q.default + 0.25 * (q.max - q.default)
            else:
                lo, hi = float(q.default - 0.25 * (q.default - q.min)), float(q.default + 0.25 * (q.max - q.default))
            narrowed.set(name, q.default, lo, hi, q.type)
        return [{"domain_rand": False}, {"domain_rand": True, "params": narrowed}, {"domain_rand": True}]

    def one(arm):
        ladder = arm == "ladder"
        kw = dict(env_level=np.zeros(args.envs, np.int32), dynamic_levels=True, level_seed=7) if ladder else {}
        env, held = build([FOURROOMS] * 3, args.envs, level_kwargs=rows(arm), **kw)
        acts = actions(env, args)
        gen = generator(env)

        def step(t):
            if ladder and t % 50 == 0:
                env.level_weights.copy_(torch.rand(3, device=acts.device, generator=gen))
            env.step(acts[t])
        rec = run(arm, env, held, args, step)
        if ladder:
            rec["envs_per_row_at_end"] = np.bincount(env.env_level, minlength=3).tolist()
        return finish(env, rec)
    return [one(arm) for _ in range(args.rounds) for arm in ("off", "on", "ladder")]


def level_params(args):
    """Cost of level params written while the batch runs (MWB_ARRAY_LEVEL_PARAMS, BatchedMiniWorld.set_level_param):
    `--envs` FourRooms envs with domain_rand on.
      * never:   the params are never written;
      * every50: every 50 steps torch ops widen or narrow forward_step's and turn_step's ranges from the rewards of the
                 last 50 steps (an automatic domain randomisation loop; no host sync);
      * every1:  the same writes before every step.
    Each run adds forward_step's range at its end."""
    import torch
    every_of = {"never": 0, "every50": 50, "every1": 1}

    def one(arm):
        every = every_of[arm]
        env, held = build(FOURROOMS, args.envs, domain_rand=True)
        acts = actions(env, args)
        dev = acts.device
        fs = torch.tensor([0.15, 0.12, 0.17], dtype=torch.float64, device=dev)
        ts = torch.tensor([15.0, 10.0, 20.0], dtype=torch.float64, device=dev)
        score = torch.zeros(args.envs, dtype=torch.float64, device=dev)

        def step(t):
            nonlocal fs, ts
            if every and t % every == 0:
                grow = torch.where(score.mean() > 0.001, 1.02, 0.99).to(torch.float64)
                fs = torch.stack([fs[0], fs[0] - (fs[0] - fs[1]) * grow, fs[0] + (fs[2] - fs[0]) * grow])
                ts = torch.stack([ts[0], ts[0] - (ts[0] - ts[1]) * grow, ts[0] + (ts[2] - ts[0]) * grow])
                env.set_level_param(0, "forward_step", fs[0], fs[1], fs[2])
                env.set_level_param(0, "turn_step", ts[0], ts[1], ts[2])
                score.zero_()
            _, rew, _, _, _ = env.step(acts[t])
            if every:
                score.add_(rew)
        rec = run(arm, env, held, args, step)
        p = env.get_level_params(0).params
        rec["forward_step_range_at_end"] = [p["forward_step"].min, p["forward_step"].max]
        return finish(env, rec)
    return [one(arm) for _ in range(args.rounds) for arm in every_of]


def maze_levels(args):
    """Cost of Maze levels in a level table (BatchedMiniWorld(levels, per_env_worlds=True)).
      * mix:         `--envs` envs over OneRoom, FourRooms, MazeS2, MazeS3 and Maze (8 x 8), contiguous blocks;
      * mix-no-maze: the same mix without Maze (what the 8 x 8 maze's HBM triangle lists cost the batch);
      * alone:       each level of the first mix alone, at its count in that mix."""
    import numpy as np
    from miniworld_b200.batched import default_env_level
    mix = ["MiniWorld-OneRoom-v0", FOURROOMS, "MiniWorld-MazeS2-v0", MAZES3, MAZE8]
    counts = np.bincount(default_env_level(args.envs, len(mix)), minlength=len(mix))

    def one(arm, levels, n):
        env, held = build(levels, n, **({} if isinstance(levels, str) else {"per_env_worlds": True}))
        acts = actions(env, args)
        rec = run(arm, env, held, args, lambda t: env.step(acts[t]))
        rec["levels"] = levels
        return finish(env, rec)

    recs = []
    for _ in range(args.rounds):
        recs.append(one("mix", mix, args.envs))
        recs.append(one("mix-no-maze", mix[:-1], int(counts[:-1].sum())))
        recs += [one("alone", lv, int(c)) for lv, c in zip(mix, counts)]
    return recs


def episode_seeds(args):
    """Cost of episode seeds (mwb_enable_episode_seeds, BatchedMiniWorld(episode_seeds=True)): `--envs` envs of
    FourRooms and of MazeS3 with truncated levels.
      * off:    episode seeds off;
      * idle:   episode seeds on, next_seed never written (every reset tests the pending seed and continues its stream);
      * replay: episode seeds on, and after every step torch ops give every done env a seed (half from a 512-seed
                buffer, half fresh), with no host sync: every reset builds a stream from its seed.
    The idle and replay runs add how many running episodes are seeded at the end."""
    import torch
    levels = {"fourrooms": FOURROOMS, "mazes3": MAZES3}

    def one(level, arm):
        n = args.envs
        env, held = build(levels[level], n, args.episode_steps, episode_seeds=arm != "off")
        acts = actions(env, args, 3)
        dev = acts.device
        gen = generator(env)
        buf_seed = torch.arange(512, device=dev)

        def step(t):
            _, _, te, tr, _ = env.step(acts[t])
            if arm == "replay":
                pick = buf_seed[torch.randint(0, 512, (n,), device=dev, generator=gen)]
                fresh = torch.randint(0, 2 ** 31, (n,), device=dev, generator=gen)
                nxt = torch.where(torch.rand(n, device=dev, generator=gen) < 0.5, pick, fresh)
                env.next_seed.copy_(torch.where(te | tr, nxt, env.next_seed))
        rec = run("%s/%s" % (level, arm), env, held, args, step)
        if arm != "off":
            rec["seeded_episodes_at_end"] = int((env.episode_seed >= 0).sum())
        return finish(env, rec)
    return [one(level, arm) for _ in range(args.rounds) for level in levels for arm in ("off", "idle", "replay")]


def maze_layouts(args):
    """Cost of maze layouts (mwb_enable_maze_layouts, BatchedMiniWorld(maze_layouts=True)): `--envs` envs of MazeS3
    and of the 8 x 8 Maze with truncated levels.
      * off:    maze layouts off (capacities sized for trees, as before);
      * idle:   maze layouts on, never written: every reset carves and records its topology, with the capacities and
                K2's lists sized for the all-open maze;
      * design: maze layouts on, and after every step torch ops give every done env an edited layout (three random
                edge bits of the layout it just played flipped, info["maze"]) and random goal / agent cells, with no
                host sync: every reset builds a designed maze and its per-env room cdf."""
    import torch
    levels = {"mazes3": MAZES3, "maze": MAZE8}

    def one(level, arm):
        n = args.envs
        env, held = build(levels[level], n, args.episode_steps, maze_layouts=arm != "off")
        acts = actions(env, args, 3)
        dev = acts.device
        gen = generator(env)
        if arm != "off":
            R, C = env.maze_shape
            rows = torch.arange(n, device=dev)

        def step(t):
            _, _, te, tr, info = env.step(acts[t])
            if arm == "design":
                done = te | tr
                lay = info["maze"].clone().view(n, R * C)
                for _ in range(3):
                    cell = torch.randint(0, R * C, (n,), device=dev, generator=gen)
                    bit = torch.randint(0, 2, (n,), device=dev, generator=gen).to(torch.uint8)
                    lay[rows, cell] ^= torch.bitwise_left_shift(torch.ones_like(bit), bit)
                cells = torch.randint(-1, R * C, (n, 2), dtype=torch.int32, device=dev, generator=gen)
                env.next_maze.copy_(torch.where(done[:, None, None], lay.view(n, R, C), env.next_maze))
                env.next_maze_cells.copy_(torch.where(done[:, None], cells, env.next_maze_cells))
                env.maze_pending.copy_(torch.where(done, torch.ones_like(env.maze_pending), env.maze_pending))
        return finish(env, run("%s/%s" % (level, arm), env, held, args, step))
    return [one(level, arm) for _ in range(args.rounds) for level in levels for arm in ("off", "idle", "design")]


def start_poses(args):
    """Cost of start poses (mwb_enable_start_poses, BatchedMiniWorld(start_poses=True)): `--envs` envs of FourRooms
    and of PickupObjects with truncated levels.
      * off:    start poses off;
      * idle:   start poses on, never written: every reset records the agent's start pose;
      * design: start poses on, and after every step torch ops give every done env a designed goal box (slot 0) and
                agent pose, drawn inside the floor plan's bounding box, with no host sync: every reset skips those
                two searches."""
    import torch
    levels = {"fourrooms": FOURROOMS, "pickup": PICKUP}

    def one(level, arm):
        n = args.envs
        env, held = build(levels[level], n, args.episode_steps, start_poses=arm != "off")
        acts = actions(env, args, 3)
        dev = acts.device
        gen = generator(env)
        rooms = env.proto_envs[0].rooms
        lo = torch.tensor([min(r.min_x for r in rooms), min(r.min_z for r in rooms)], dtype=torch.float64, device=dev)
        hi = torch.tensor([max(r.max_x for r in rooms), max(r.max_z for r in rooms)], dtype=torch.float64, device=dev)

        def step(t):
            _, _, te, tr, _ = env.step(acts[t])
            if arm == "design":
                done = (te | tr)[:, None]
                goal = lo + torch.rand((n, 2), dtype=torch.float64, device=dev, generator=gen) * (hi - lo)
                agent = lo + torch.rand((n, 2), dtype=torch.float64, device=dev, generator=gen) * (hi - lo)
                env.next_pose[:, 0, :2] = torch.where(done, goal, env.next_pose[:, 0, :2])
                env.next_agent_pose[:, :2] = torch.where(done, agent, env.next_agent_pose[:, :2])
                env.pose_pending.copy_(torch.where(done[:, 0], torch.ones_like(env.pose_pending), env.pose_pending))
        return finish(env, run("%s/%s" % (level, arm), env, held, args, step))
    return [one(level, arm) for _ in range(args.rounds) for level in levels for arm in ("off", "idle", "design")]


def reset_draws(args):
    """Cost of reset draws (mwb_enable_reset_draws, BatchedMiniWorld(reset_draws=True)): `--envs` envs of
    PickupObjects and of TMaze with truncated levels.
      * off:    reset draws off;
      * idle:   reset draws on, never written: every reset records the outcome of each of its draws;
      * design: reset draws on, and after every step torch ops give every done env a design for every draw, drawn
                inside the draw's support (PickupObjects: kinds and colours of its five objects; TMaze: goal side and
                heading), with no host sync."""
    import torch
    levels = {"pickup": PICKUP, "tmaze": "MiniWorld-TMaze-v0"}

    def one(level, arm):
        n = args.envs
        env, held = build(levels[level], n, args.episode_steps, reset_draws=arm != "off")
        acts = actions(env, args, 3)
        dev = acts.device
        gen = generator(env)
        # each draw's support as (lo, width): a choice over n draws floor(n u), a uniform lo + (hi - lo) u
        specs = env.draw_specs[0]
        lo = torch.tensor([0.0 if s["kind"] == "choice" else s["lo"] for s in specs], dtype=torch.float64, device=dev)
        width = torch.tensor([s["n"] if s["kind"] == "choice" else s["hi"] - s["lo"] for s in specs],
                             dtype=torch.float64, device=dev)
        choice = torch.tensor([s["kind"] == "choice" for s in specs], device=dev)

        def step(t):
            _, _, te, tr, _ = env.step(acts[t])
            if arm == "design":
                done = te | tr
                u = lo + torch.rand((n, len(specs)), dtype=torch.float64, device=dev, generator=gen) * width
                design = torch.where(choice, torch.floor(u), u)
                env.next_draws.copy_(torch.where(done[:, None], design, env.next_draws))
                env.draws_pending.copy_(torch.where(done, torch.ones_like(env.draws_pending), env.draws_pending))
        return finish(env, run("%s/%s" % (level, arm), env, held, args, step))
    return [one(level, arm) for _ in range(args.rounds) for level in levels for arm in ("off", "idle", "design")]


def env_params(args):
    """Cost of env params (mwb_enable_env_params, BatchedMiniWorld(env_params=True)): `--envs` envs of FourRooms and
    of PickupObjects with domain randomisation and truncated levels.
      * off:  env params off;
      * idle: env params on, never written: every reset writes a NaN row, every step merges nothing;
      * adr:  env params on, and after every step the README's ADR loop in torch ops gives every done env a design
              (with probability 0.5 one random element pinned at its level's lower or upper bound, otherwise an
              all-NaN row), with no host sync.
    Then the same rounds run again under torch.profiler (CUDA activity only, no timing of their own) for K1's device
    time per launch."""
    import torch
    from miniworld_b200.engine import ENV_PARAM_ELEMS, PARAMS_COLUMN
    levels = {"fourrooms": FOURROOMS, "pickup": PICKUP}
    arms = ("off", "idle", "adr")

    def adr_update(env, done, gen):
        """The README ADR step: each done env pins one random element at its level's current lower or upper bound
        with probability 0.5, otherwise gets an all-NaN row; both set the pending flag."""
        n, dev = env.num_envs, done.device
        lp = env._views()["level_params"][0]
        e = torch.randint(0, ENV_PARAM_ELEMS, (n,), device=dev, generator=gen)
        upper = torch.rand(n, device=dev, generator=gen) < 0.5
        probe = done & (torch.rand(n, device=dev, generator=gen) < 0.5)
        word = torch.where(e < 15, (e // 3) * 9 + e % 3, 45 + (e - 15) * 3)     # the element's default in mwb_params
        step = torch.where(e < 15, 3, 1)
        lo = lp[word + step]
        hi = torch.where(e == 15, lp[PARAMS_COLUMN["max_forward_step"]], lo + lp[word + 2 * step])
        row = torch.full((n, ENV_PARAM_ELEMS, 3), float("nan"), dtype=torch.float64, device=dev)
        row[probe, e[probe]] = torch.where(upper, hi, lo)[probe].unsqueeze(1).expand(-1, 3)
        env.next_params.copy_(torch.where(done[:, None, None], row, env.next_params))
        env.params_pending.copy_(torch.where(done, torch.ones_like(env.params_pending), env.params_pending))

    def setup(level, arm):
        env, held = build(levels[level], args.envs, args.episode_steps, domain_rand=True, env_params=arm != "off")
        acts = actions(env, args, 3)
        gen = generator(env)

        def step(t):
            _, _, te, tr, _ = env.step(acts[t])
            if arm == "adr":
                adr_update(env, te | tr, gen)
        return env, held, step

    def one(level, arm):
        env, held, step = setup(level, arm)
        return finish(env, run("%s/%s" % (level, arm), env, held, args, step))

    def profiled(level, arm):
        env, _, step = setup(level, arm)
        for t in range(args.warmup):
            step(t)
        torch.cuda.synchronize()
        ms, count = kernel_ms(lambda: [step(t) for t in range(args.warmup, args.warmup + args.steps)],
                              ("step_kernel",)).get("step_kernel", (0.0, 0))
        return finish(env, {"arm": "%s/%s" % (level, arm), "profiler": "torch", "k1_launches": count,
                            "k1_us_per_launch": ms * 1e3 / max(count, 1)})
    return [f(level, arm) for f in (one, profiled) for _ in range(args.rounds) for level in levels for arm in arms]


def state_bank(args):
    """Cost of the state bank (mwb_enable_state_bank, BatchedMiniWorld(state_bank=K)): `--envs` envs of FourRooms,
    MazeS3 and the 8 x 8 Maze with truncated levels.
      * off:     no state bank;
      * idle:    a bank of `--slots` slots, never written: every reset reads next_state and writes episode_state;
      * explore: after every step torch ops save about 5 % of the envs into random slots and give every done env a
                 pending slot drawn from the filled ones, with no host sync: most resets load a record instead of
                 running the level's program.
    The runs with a bank add the device memory per slot (against the off arm of the same round) and, for explore,
    how many running episodes started from a record.  After the rounds, saves of all envs (one mwb_save_states call,
    `--envs` distinct slots) are timed with CUDA events over 50 calls per level, with the bytes a save must move
    (read the env's rows and the world in use, write the record) over that time, against the 3.35 TB/s HBM3 figure of
    the H100 SXM data sheet."""
    import torch
    levels = {"fourrooms": FOURROOMS, "mazes3": MAZES3, "maze8": MAZE8}
    off_held = {}

    def one(level, arm):
        n, slots = args.envs, args.slots
        env, held = build(levels[level], n, args.episode_steps, state_bank=None if arm == "off" else slots)
        acts = actions(env, args, 3)
        dev = acts.device
        gen = generator(env)
        k = max(1, n // 20)

        def step(t):
            _, _, te, tr, _ = env.step(acts[t])
            if arm == "explore":
                who = torch.randint(0, n, (k,), device=dev, generator=gen)
                env.save_states(who, torch.randint(0, slots, (k,), device=dev, generator=gen))
                cdf = (env.bank_level >= 0).long().cumsum(0)
                u = (torch.rand(n, generator=gen, device=dev, dtype=torch.float64) * cdf[-1]).long()
                pick = torch.searchsorted(cdf, u, right=True).clamp(max=slots - 1)
                env.next_state.copy_(torch.where(te | tr, pick, -1).int())
        rec = run("%s/%s" % (level, arm), env, held, args, step)
        if arm == "off":
            off_held[level] = held
        else:
            rec.update(slots=slots, device_bytes_per_slot=(held - off_held[level]) / slots)
            if arm == "explore":
                rec["loaded_episodes_running"] = int((env.episode_state >= 0).sum())
        return finish(env, rec)

    def save_all(level, calls=50):
        from miniworld_b200.batched import BatchedMiniWorld
        n = args.envs
        env = BatchedMiniWorld(short_level(levels[level], args.episode_steps), n, state_bank=n)
        env.reset(seed=7)
        ids = torch.arange(n, device="cuda", dtype=torch.int32)
        slots = torch.randperm(n, device="cuda").int()
        for _ in range(5):
            env.save_states(ids, slots)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            env.save_states(ids, slots)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / calls
        # the scalar part of a record from the field sizes (264 B + 68 B per entity slot + 12 B per room), and the
        # mean bytes of the world in use of the first 64 envs (0 when the level has no per-env worlds)
        scalar = 264 + 68 * env.engine.max_ents + 12 * env.engine.cfg.max_rooms
        world = 0.0 if env.maze_template is None else sum(
            sum(a.nbytes for a in env.engine.get_geometry(i)) for i in range(min(64, n))) / min(64, n)
        moved = 2.0 * n * (scalar + world)       # read the env's rows, write the record
        return finish(env, {"arm": "%s/save_all" % level, "envs": n, "ms_per_call": ms, "bytes_moved": moved,
                            "scalar_bytes_per_record": scalar, "world_bytes_in_use_per_env": world,
                            "achieved_bytes_per_s": moved / (ms * 1e-3),
                            "share_of_hbm_3_35TBps": moved / (ms * 1e-3) / 3.35e12})

    names = args.levels.split(",")
    recs = [one(level, arm) for _ in range(args.rounds) for level in names for arm in ("off", "idle", "explore")]
    return recs + [save_all(level) for level in names]


def goal_distance(args):
    """Cost of goal distance (mwb_enable_goal_distance, BatchedMiniWorld(goal_distance=True)): `--envs` envs of
    FourRooms, MazeS3 and the 8 x 8 Maze with truncated levels.
      * off:    goal distance off, random actions;
      * random: goal distance on, random actions;
      * expert: goal distance on, every step's actions are the previous step's expert_action (no host sync).
    The runs with the mode on add the grid size next to the 3 G + 21 bytes the arrays take per env, the share of steps
    whose goal_dist is +inf, the goal distance kernel's and K1's time per launch from torch.profiler (a separate,
    shorter window), and a reset of all envs timed on its own: the goal distance kernel's time then is the field build
    of every env, reported per env."""
    import torch
    levels = {"fourrooms": FOURROOMS, "mazes3": MAZES3, "maze8": MAZE8}

    def one(level, arm):
        n = args.envs
        env, held = build(levels[level], n, args.episode_steps, goal_distance=arm != "off")
        acts = actions(env, args, 3)
        dev = acts.device
        unreached = torch.zeros((), dtype=torch.int64, device=dev)
        expert = torch.zeros(n, dtype=torch.int32, device=dev)

        def step(t):
            if arm == "expert":
                expert.copy_(env.expert_action.clamp(0, 2))
            env.step(expert if arm == "expert" else acts[t])
            if arm != "off":
                unreached.add_(torch.isinf(env.goal_dist).sum())
        rec = run("%s/%s" % (level, arm), env, held, args, step, at_start=unreached.zero_)
        if arm != "off":
            G = env.goal_field.shape[1]
            rec.update(grid_nodes=G, goal_distance_bytes_per_env=3 * G + 21,
                       unreachable_share=int(unreached) / (n * args.steps))
            window = min(args.steps, 50)
            times = kernel_ms(lambda: [step(t) for t in range(args.warmup, args.warmup + window)],
                              ("nav_kernel", "step_kernel"))
            nav, k1 = times.get("nav_kernel", (float("nan"), 1)), times.get("step_kernel", (float("nan"), 1))
            rec["nav_ms_per_launch"] = nav[0] / max(nav[1], 1)
            rec["k1_profiled_ms_per_launch"] = k1[0] / max(k1[1], 1)
            # a reset of every env: the goal distance kernel then builds all n fields (CUDA events around the call,
            # which launches reset_kernel and the goal distance kernel; the profiler splits the two where it records
            # both)
            stream = torch.cuda.current_stream(dev)
            r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            r0.record()
            env.engine.reset(stream=stream.cuda_stream or 1)
            r1.record()
            torch.cuda.synchronize()
            rec["full_reset_ms"] = r0.elapsed_time(r1)
            full = kernel_ms(lambda: env.engine.reset(stream=stream.cuda_stream or 1), ("nav_kernel", "reset_kernel"))
            rec["full_reset_nav_ms"] = full.get("nav_kernel", (float("nan"), 0))[0]
            rec["field_build_us_per_env"] = rec["full_reset_nav_ms"] * 1e3 / n
            rec["full_reset_kernel_ms"] = full.get("reset_kernel", (float("nan"), 0))[0]
        return finish(env, rec)
    return [one(level, arm) for _ in range(args.rounds) for level in levels for arm in ("off", "random", "expert")]


def views(args):
    """Cost of designed-camera views (mwb_render_views, BatchedMiniWorld.render_views): `--envs` envs of FourRooms and
    of PickupObjects with truncated levels.
      * step:  step only;
      * full:  step, then one view of every env from a row written by torch ops (1.5 m from the agent, facing it);
      * done:  step, then the ImageNav goal image: views only for the envs that just ended, every other row NaN
               (skipped);
      * pano:  step, then a four-heading panorama of every env (V = 4 views 90 degrees apart at the agent's position).
    Each run adds the time of the render_views calls alone (CUDA events around them) per call and per view; the K2
    average covers the step's observation launch and the view launches.  The step runs add the time of an
    all-skipped call (every row NaN, one view) over 200 calls: the floor a skipped view costs."""
    import torch
    levels = {"fourrooms": FOURROOMS, "pickup": PICKUP}

    def one(level, arm):
        n = args.envs
        env, held = build(levels[level], n, args.episode_steps)
        acts = actions(env, args, 3)
        dev = acts.device
        slot = [s["slot"] for s in env.level_slots[0] if s["agent"]][0]
        nviews = 4 if arm == "pano" else 1
        out = torch.zeros((nviews,) + env.obs_shape, dtype=torch.uint8, device=dev)
        nan = torch.full((n, 3), math.nan, dtype=torch.float64, device=dev)
        quarter = torch.arange(4, device=dev, dtype=torch.float64)[:, None] * (math.pi / 2)
        ev = []

        def rows(done):
            xz = env.entity_xz(slot)
            d = env._views()["ent_dir"][slot]
            if arm == "pano":
                return torch.stack([torch.cat([xz, (d[None] + quarter[k]).T], 1) for k in range(4)])
            eye = xz - 1.5 * torch.stack([d.cos(), -d.sin()], 1)        # 1.5 m behind the agent, facing it
            r = torch.cat([eye, d[:, None]], 1)
            return torch.where(done[:, None], r, nan) if arm == "done" else r

        def step(t):
            _, _, te, tr, _ = env.step(acts[t])
            if arm == "step":
                return
            r = rows(te | tr)
            timed = t >= args.warmup
            if timed:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
            env.render_views(r, out=out if arm == "pano" else out[0])
            if timed:
                b.record()
                ev.append((a, b))
        rec = run("%s/%s" % (level, arm), env, held, args, step)
        view_ms = sum(a.elapsed_time(b) for a, b in ev) / max(len(ev), 1)
        rec.update(views_ms_per_call=view_ms, views_ms_per_view=view_ms / nviews)
        if arm == "step":                      # the floor of a skipped view: one all-NaN view, 200 calls
            for _ in range(20):
                env.render_views(nan, out=out[0])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(200):
                env.render_views(nan, out=out[0])
            e1.record()
            torch.cuda.synchronize()
            rec["all_skipped_ms_per_call"] = e0.elapsed_time(e1) / 200
        return finish(env, rec)
    return [one(level, arm) for _ in range(args.rounds) for level in levels for arm in ("step", "full", "done", "pano")]


def view_cameras(args):
    """Cost of designed cameras with their own intrinsics, frame size and sample count (7-column rows,
    BatchedMiniWorld.render_views(size=, samples=)): `--envs` envs of FourRooms and of PickupObjects with truncated
    levels, mwb_profile off.
      * step:   step only;
      * rows3:  step, then one 80x60/8 view per env from 3-column rows (1.5 m behind the agent, facing its heading);
      * rows7:  the same rows as 7-column rows with every intrinsic NaN (the same frames);
      * chase:  step, then a chase view per env at 160x120/16: 3 m behind the agent, 2.5 m up, pitched -25 degrees,
                marker drawn;
      * twocam: step, then a two-camera observation at 80x60/8 (FOV 110 and FOV 40 at the agent's eye).
    Each run adds the time of the render_views calls alone (CUDA events around them) per call.  After the arms of a
    level in each round: the first call at a new frame size (160x120/16 on a fresh batch; staging allocation and the
    shared-memory opt-in) against the mean of the next 50 calls, host clock around work that ends in a device
    synchronise."""
    import torch
    levels = {"fourrooms": FOURROOMS, "pickup": PICKUP}
    arms = ("step", "rows3", "rows7", "chase", "twocam")

    def one(level, arm):
        n = args.envs
        env, held = build(levels[level], n, args.episode_steps)
        acts = actions(env, args, 3)
        dev = acts.device
        slot = [s["slot"] for s in env.level_slots[0] if s["agent"]][0]
        size, samples, nviews = ((160, 120), 16, 1) if arm == "chase" else ((80, 60), 8, 2 if arm == "twocam" else 1)
        out = torch.zeros((nviews, n, size[1], size[0], 3), dtype=torch.uint8, device=dev)
        r7 = torch.full((nviews, n, 7), math.nan, dtype=torch.float64, device=dev)
        if arm == "chase":
            r7[0, :, 3:6] = torch.tensor([2.5, 0.0, -25.0], dtype=torch.float64)
        if arm == "twocam":
            r7[0, :, 6], r7[1, :, 6] = 110.0, 40.0
        ev = []

        def rows():
            xz = env.entity_xz(slot)
            d = env._views()["ent_dir"][slot]
            back = 3.0 if arm == "chase" else (0.0 if arm == "twocam" else 1.5)
            r7[:, :, :2] = xz - back * torch.stack([d.cos(), -d.sin()], 1)
            r7[:, :, 2] = d
            return r7[0, :, :3].contiguous() if arm == "rows3" else (r7 if nviews > 1 else r7[0])

        def step(t):
            env.step(acts[t])
            if arm == "step":
                return
            r = rows()
            timed = t >= args.warmup
            if timed:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
            env.render_views(r, render_agent=arm == "chase", out=out if nviews > 1 else out[0], size=size,
                             samples=samples)
            if timed:
                b.record()
                ev.append((a, b))
        rec = run("%s/%s" % (level, arm), env, held, args, step, profile=False)
        rec["views_ms_per_call"] = sum(a.elapsed_time(b) for a, b in ev) / max(len(ev), 1)
        return finish(env, rec)

    def first_call(level):
        from miniworld_b200.batched import BatchedMiniWorld
        n = args.envs
        env = BatchedMiniWorld(levels[level], n)
        env.reset(seed=7)
        env.render_views(torch.full((n, 3), math.nan, dtype=torch.float64, device="cuda"))     # module and 80x60 warm
        st = env.get_state()
        r = torch.tensor([[p[0], p[2], d, 2.5, 0.0, -25.0, math.nan] for p, d in zip(st["agent_pos"], st["agent_dir"])],
                         dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = env.render_views(r, size=(160, 120), samples=16)
        torch.cuda.synchronize()
        first = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        for _ in range(50):
            env.render_views(r, out=out, size=(160, 120), samples=16)
        torch.cuda.synchronize()
        later = (time.perf_counter() - t0) * 1e3 / 50
        return finish(env, {"arm": "%s/first_call_160x120x16" % level, "first_ms": first, "later_ms": later})
    return [rec for _ in range(args.rounds) for level in levels
            for rec in [one(level, arm) for arm in arms] + [first_call(level)]]


STUDIES = {f.__name__: f for f in (configs, mixed, level_changes, level_dr, level_params, maze_levels, episode_seeds,
                                   maze_layouts, start_poses, reset_draws, env_params, state_bank, goal_distance, views,
                                   view_cameras)}
TRUNCATED = ("episode_seeds", "maze_layouts", "start_poses", "reset_draws", "env_params", "state_bank", "goal_distance",
             "views", "view_cameras")


def parse_args():
    raw = argparse.RawDescriptionHelpFormatter
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=raw)
    sub = ap.add_subparsers(dest="study", required=True, metavar="STUDY", help=", ".join(STUDIES))
    for name, fn in STUDIES.items():
        p = sub.add_parser(name, description=inspect.cleandoc(fn.__doc__), formatter_class=raw)
        if name != "configs":            # configs runs each config at its own env count
            p.add_argument("--envs", type=int, default=4096)
        p.add_argument("--steps", type=int, default=100 if name == "configs" else 200)
        p.add_argument("--warmup", type=int, default=10 if name == "configs" else 20)
        p.add_argument("--rounds", type=int, default=1 if name in ("configs", "mixed") else 3)
        if name in TRUNCATED:
            p.add_argument("--episode-steps", type=int, default=20)
        if name in ("mixed", "level_changes"):
            p.add_argument("--levels", nargs="+", default=MIX4, metavar="ID")
        if name == "state_bank":
            p.add_argument("--levels", default="fourrooms,mazes3,maze8")
            p.add_argument("--slots", type=int, default=4096)
        p.add_argument("--baseline-tree", metavar="DIR", help="built checkout of the revision to compare bench.py against")
        p.add_argument("--bench-steps", type=int, default=200)
        p.add_argument("--bench-warmup", type=int, default=20)
        p.add_argument("--bench-only", action="store_true", help="skip part 1")
    return ap.parse_args()


def main():
    args = parse_args()
    print(json.dumps(card()), flush=True)
    if not args.bench_only:
        summary(STUDIES[args.study](args))
    if args.baseline_tree:
        compare_trees(args)


if __name__ == "__main__":
    main()
