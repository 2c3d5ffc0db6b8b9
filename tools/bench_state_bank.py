"""Cost of the state bank (mwb_enable_state_bank, BatchedMiniWorld(state_bank=K)), measured on one GPU.

    python tools/bench_state_bank.py [--envs 4096] [--slots 4096] [--steps 200] [--warmup 20] [--rounds 3]
                                     [--episode-steps 20] [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20]

Part 1: 4096 envs of FourRooms, MazeS3 and the 8 x 8 Maze, device-resident like bench.py's main arm, with episodes
truncated after `--episode-steps` steps so that a twentieth of the envs reset in every step.  Three arms run
alternately for `--rounds` rounds:
  * off:     no state bank;
  * idle:    a bank of `--slots` slots, never written: every reset reads next_state and writes episode_state;
  * explore: after every step torch ops save about 5 % of the envs into random slots and give every done env a pending
             slot drawn from the filled ones, with no host sync: most resets load a record instead of running the
             level's program.
Each run prints one JSON line (env-steps/s from CUDA events, K1 / K2 time per launch from mwb_profile, the device
memory the batch holds per env and, with the bank, per slot, from cudaMemGetInfo around its construction, against the
off arm of the same round); a summary line per level and arm gives the median and the spread (min, max) over the rounds.

Part 2: saves of all envs (one mwb_save_states call, 4096 distinct slots) timed with CUDA events over 50 calls per
level, with the bytes a save must move (read the env's rows and the world in use, write the record) over that time,
against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet.

Part 3 (with `--baseline-tree DIR`, a built checkout of another revision): `bench.py --gpus 1` (default config) and
`bench.py --gpus 1 --config 4` of DIR and of this tree, alternately, `--rounds` times each, then `--dump-outputs` of
both compared file by file (tools/bench_level_dr.py's part 2).
The first line names the card and its power limit.  Nothing is written to either tree.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_level_changes import card  # noqa: E402
from bench_level_dr import run_bench, same_dumps, summary  # noqa: E402
from bench_start_poses import short_level  # noqa: E402

LEVELS = {"fourrooms": "MiniWorld-FourRooms-v0", "mazes3": "MiniWorld-MazeS3-v0", "maze8": "MiniWorld-Maze-v0"}
ARMS = ("off", "idle", "explore")
HBM_BYTES_PER_S = 3.35e12


def world_bytes(env, sample=64):
    """Mean bytes of the world in use of the first `sample` envs (0 when the level has no per-env worlds)."""
    if env.maze_template is None:
        return 0.0
    tot = 0
    for i in range(min(sample, env.num_envs)):
        rooms, quads, segs = env.engine.get_geometry(i)
        tot += rooms.nbytes + quads.nbytes + segs.nbytes
    return tot / min(sample, env.num_envs)


def scalar_bytes(env):
    """The scalar part of a record, from the field sizes: 264 B + 68 B per entity slot + 12 B per room."""
    return 264 + 68 * env.engine.max_ents + 12 * env.engine.cfg.max_rooms


def run_arm(level, arm, n, slots, steps, warmup, episode_steps, free_off=None):
    import numpy as np
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    dev = torch.device("cuda", 0)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    env = BatchedMiniWorld(short_level(LEVELS[level], episode_steps), n, state_bank=None if arm == "off" else slots)
    env.reset(seed=1000)
    torch.cuda.synchronize()
    held = free0 - torch.cuda.mem_get_info(dev)[0]
    acts = torch.as_tensor(np.random.default_rng(12345).integers(0, 3, size=(warmup + steps, n), dtype=np.int32), device=dev)
    stagger = torch.as_tensor(env.engine.state_array("step_count"), device=dev)
    stagger.copy_(torch.arange(n, device=dev, dtype=torch.int32) % episode_steps)
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)
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

    for t in range(warmup):
        step(t)
    torch.cuda.synchronize()
    env.engine.profile(True)
    env.engine.profile_read()
    done0 = int(env.get_state()["episodes_done"][0])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(warmup, warmup + steps):
        step(t)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    k1, k2, n1, n2 = env.engine.profile_read()
    env.engine.profile(False)
    assert env.engine.overflow_count() == 0
    rec = {"arm": "%s/%s" % (level, arm), "envs": n, "steps": steps, "env_steps_per_s": n * steps / (ms * 1e-3),
           "ms_per_step": ms / steps, "k1_ms_per_launch": k1 / max(n1, 1), "k2_ms_per_launch": k2 / max(n2, 1),
           "resets_per_step": (int(env.get_state()["episodes_done"][0]) - done0) / steps,
           "device_bytes_per_env": held / n}
    if arm != "off":
        rec["slots"] = slots
        if free_off is not None:
            rec["device_bytes_per_slot"] = (held - free_off) / slots
        if arm == "explore":
            rec["loaded_episodes_running"] = int((env.episode_state >= 0).sum())
    env.close()
    print(json.dumps(rec), flush=True)
    return rec, held


def time_saves(level, n, episode_steps, calls=50):
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    dev = torch.device("cuda", 0)
    env = BatchedMiniWorld(short_level(LEVELS[level], episode_steps), n, state_bank=n)
    env.reset(seed=7)
    ids = torch.arange(n, device=dev, dtype=torch.int32)
    slots = torch.randperm(n, device=dev).int()
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
    moved = 2.0 * n * (scalar_bytes(env) + world_bytes(env))       # read the env's rows, write the record
    rec = {"arm": "%s/save_all" % level, "envs": n, "ms_per_call": ms, "bytes_moved": moved,
           "scalar_bytes_per_record": scalar_bytes(env), "world_bytes_in_use_per_env": world_bytes(env),
           "achieved_bytes_per_s": moved / (ms * 1e-3), "share_of_hbm_3_35TBps": moved / (ms * 1e-3) / HBM_BYTES_PER_S}
    env.close()
    print(json.dumps(rec), flush=True)
    return rec


def main():
    import tempfile
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--slots", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--episode-steps", type=int, default=20)
    ap.add_argument("--levels", default=",".join(LEVELS))
    ap.add_argument("--baseline-tree", metavar="DIR", help="built checkout of the revision to compare bench.py against")
    ap.add_argument("--bench-steps", type=int, default=200)
    ap.add_argument("--bench-warmup", type=int, default=20)
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    levels = args.levels.split(",")
    recs = []
    for _ in range(args.rounds):
        for level in levels:
            off = None
            for arm in ARMS:
                rec, held = run_arm(level, arm, args.envs, args.slots, args.steps, args.warmup, args.episode_steps, off)
                off = held if arm == "off" else off
                recs.append(rec)
    summary(recs)
    for level in levels:
        time_saves(level, args.envs, args.episode_steps)
    if not args.baseline_tree:
        return
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
            names, same = same_dumps(a, b)
            print(json.dumps({"arm": "dump-outputs", "config": config or "default", "files": names,
                              "byte_identical": same}), flush=True)


if __name__ == "__main__":
    main()
