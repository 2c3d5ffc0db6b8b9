"""Cost of goal distance (mwb_enable_goal_distance, BatchedMiniWorld(goal_distance=True)), measured on one GPU.

    python tools/bench_goal_distance.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3] [--episode-steps 20]
                                        [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20]

Part 1: 4096 envs of FourRooms, MazeS3 and the 8 x 8 Maze, device-resident like bench.py's main arm, with episodes
truncated after `--episode-steps` steps so that a twentieth of the envs reset in every step.  Three arms run alternately
for `--rounds` rounds:
  * off:    goal distance off, random actions;
  * random: goal distance on, random actions;
  * expert: goal distance on, every step's actions are the previous step's expert_action (no host sync).
Each run prints one JSON line: env-steps/s from CUDA events, K1 / K2 time per launch from mwb_profile, the goal
distance kernel's time per launch from torch.profiler (a separate, shorter window), the device memory the batch holds
per env (cudaMemGetInfo around its construction) next to the 3 G + 21 bytes the arrays take, and for the arms with the
mode on the share of steps whose goal_dist is +inf.  A reset of all envs is profiled on its own: the goal distance
kernel's time then is the field build of every env, reported per env.  A summary line per level and arm gives the
median and the spread (min, max) over the rounds.

Part 2 (with `--baseline-tree DIR`, a built checkout of another revision): `bench.py --gpus 1` (default config) and
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
from bench_reset_draws import short_level  # noqa: E402

LEVELS = {"fourrooms": "MiniWorld-FourRooms-v0", "mazes3": "MiniWorld-MazeS3-v0", "maze8": "MiniWorld-Maze-v0"}
ARMS = ("off", "random", "expert")


def kernel_ms(fn, names):
    """Device time (ms) per name of the kernels whose names contain it, over one call of fn, with launch counts."""
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


def run_arm(level, arm, n, steps, warmup, episode_steps):
    import numpy as np
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    dev = torch.device("cuda", 0)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    env = BatchedMiniWorld(short_level(LEVELS[level], episode_steps), n, goal_distance=arm != "off")
    env.reset(seed=1000)
    torch.cuda.synchronize()
    bytes_per_env = (free0 - torch.cuda.mem_get_info(dev)[0]) / n
    acts = torch.as_tensor(np.random.default_rng(12345).integers(0, 3, size=(warmup + steps, n), dtype=np.int32), device=dev)
    # staggered starts, so that the resets spread over the steps instead of all falling into one
    stagger = torch.as_tensor(env.engine.state_array("step_count"), device=dev)
    stagger.copy_(torch.arange(n, device=dev, dtype=torch.int32) % episode_steps)
    unreached = torch.zeros((), dtype=torch.int64, device=dev)
    expert = torch.zeros(n, dtype=torch.int32, device=dev)

    def step(t):
        if arm == "expert":
            expert.copy_(env.expert_action.clamp(0, 2))
        env.step(expert if arm == "expert" else acts[t])
        if arm != "off":
            unreached.add_(torch.isinf(env.goal_dist).sum())

    for t in range(warmup):
        step(t)
    torch.cuda.synchronize()
    unreached.zero_()
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
    resets = (int(env.get_state()["episodes_done"][0]) - done0) / steps
    rec = {"arm": "%s/%s" % (level, arm), "envs": n, "steps": steps, "env_steps_per_s": n * steps / (ms * 1e-3),
           "ms_per_step": ms / steps, "k1_ms_per_launch": k1 / max(n1, 1), "k2_ms_per_launch": k2 / max(n2, 1),
           "resets_per_step": resets, "device_bytes_per_env": bytes_per_env}
    if arm != "off":
        G = env.goal_field.shape[1]
        rec.update(grid_nodes=G, goal_distance_bytes_per_env=3 * G + 21,
                   unreachable_share=int(unreached) / (n * steps))
        window = min(steps, 50)
        times = kernel_ms(lambda: [step(t) for t in range(warmup, warmup + window)], ("nav_kernel", "step_kernel"))
        nav, k1 = times.get("nav_kernel", (float("nan"), 1)), times.get("step_kernel", (float("nan"), 1))
        rec["nav_ms_per_launch"] = nav[0] / max(nav[1], 1)
        rec["k1_profiled_ms_per_launch"] = k1[0] / max(k1[1], 1)
        # a reset of every env: the goal distance kernel then builds all n fields (CUDA events around the call, which
        # launches reset_kernel and the goal distance kernel; the profiler splits the two where it records both)
        stream = torch.cuda.current_stream(dev)
        r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        r0.record()
        env.engine.reset(stream=stream.cuda_stream or 1)
        r1.record()
        torch.cuda.synchronize()
        rec["full_reset_ms"] = r0.elapsed_time(r1)
        full = kernel_ms(lambda: env.engine.reset(stream=stream.cuda_stream or 1), ("nav_kernel", "reset_kernel"))
        nav_ms = full.get("nav_kernel", (float("nan"), 0))[0]
        rec["full_reset_nav_ms"] = nav_ms
        rec["field_build_us_per_env"] = nav_ms * 1e3 / n
        rec["full_reset_kernel_ms"] = full.get("reset_kernel", (float("nan"), 0))[0]
    assert env.engine.overflow_count() == 0
    env.close()
    print(json.dumps(rec), flush=True)
    return rec


def main():
    import tempfile
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--episode-steps", type=int, default=20)
    ap.add_argument("--baseline-tree", metavar="DIR", help="built checkout of the revision to compare bench.py against")
    ap.add_argument("--bench-steps", type=int, default=200)
    ap.add_argument("--bench-warmup", type=int, default=20)
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    recs = []
    for _ in range(args.rounds):
        for level in LEVELS:
            for arm in ARMS:
                recs.append(run_arm(level, arm, args.envs, args.steps, args.warmup, args.episode_steps))
    summary(recs)
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
