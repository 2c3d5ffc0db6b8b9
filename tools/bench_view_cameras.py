"""Cost of designed cameras with their own intrinsics, frame size and sample count (7-column rows,
BatchedMiniWorld.render_views(size=, samples=)), measured on one GPU.

    python tools/bench_view_cameras.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3] [--episode-steps 20]
                                       [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20] [--bench-only]

Part 1: 4096 envs of FourRooms and of PickupObjects, device-resident like bench.py's main arm, episodes truncated after
`--episode-steps` steps (staggered).  Arms, run alternately for `--rounds` rounds:
  * step:   step only;
  * rows3:  step, then one 80x60/8 view per env from 3-column rows (1.5 m behind the agent, facing its heading);
  * rows7:  the same rows as 7-column rows with every intrinsic NaN (the same frames);
  * chase:  step, then a chase view per env at 160x120/16: 3 m behind the agent, 2.5 m up, pitched -25 degrees, marker
            drawn;
  * twocam: step, then a two-camera observation at 80x60/8 (FOV 110 and FOV 40 at the agent's eye).
Each run prints one JSON line: env-steps/s from CUDA events and the time of the render_views calls alone (CUDA events
around them) per call.  After the arms, per level: the first call at a new frame size (160x120/16 on a fresh batch;
staging allocation and the shared-memory opt-in) against the mean of the next 50 calls, host clock around work that
ends in a device synchronise.  A summary line per level and arm gives the median and the spread (min, max).

Part 2 (with `--baseline-tree DIR`, a built checkout of another revision): bench.py default and `--config 4` of DIR and
of this tree, alternately, `--rounds` times each, then `--dump-outputs` of both compared file by file.
The first line names the card and its power limit.  Nothing is written to either tree.
"""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_level_changes import card  # noqa: E402
from bench_level_dr import run_bench, same_dumps, summary  # noqa: E402
from bench_reset_draws import short_level  # noqa: E402

LEVELS = {"fourrooms": "MiniWorld-FourRooms-v0", "pickup": "MiniWorld-PickupObjects-v0"}
ARMS = ("step", "rows3", "rows7", "chase", "twocam")


def run_arm(level, arm, n, steps, warmup, episode_steps):
    import numpy as np
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    dev = torch.device("cuda", 0)
    env = BatchedMiniWorld(short_level(LEVELS[level], episode_steps), n)
    env.reset(seed=1000)
    acts = torch.as_tensor(np.random.default_rng(12345).integers(0, 3, size=(warmup + steps, n), dtype=np.int32), device=dev)
    stagger = torch.as_tensor(env.engine.state_array("step_count"), device=dev)
    stagger.copy_(torch.arange(n, device=dev, dtype=torch.int32) % episode_steps)
    slot = [s["slot"] for s in env.level_slots[0] if s["agent"]][0]
    size, samples, views = ((160, 120), 16, 1) if arm == "chase" else ((80, 60), 8, 2 if arm == "twocam" else 1)
    out = torch.zeros((views, n, size[1], size[0], 3), dtype=torch.uint8, device=dev)
    r7 = torch.full((views, n, 7), math.nan, dtype=torch.float64, device=dev)
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
        return r7[0, :, :3].contiguous() if arm == "rows3" else (r7 if views > 1 else r7[0])

    def step(t, timed):
        env.step(acts[t])
        if arm == "step":
            return
        r = rows()
        if timed:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
        env.render_views(r, render_agent=arm == "chase", out=out if views > 1 else out[0], size=size, samples=samples)
        if timed:
            b.record()
            ev.append((a, b))

    for t in range(warmup):
        step(t, False)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(warmup, warmup + steps):
        step(t, True)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    view_ms = sum(a.elapsed_time(b) for a, b in ev) / max(len(ev), 1)
    assert env.engine.overflow_count() == 0
    env.close()
    rec = {"arm": "%s/%s" % (level, arm), "envs": n, "steps": steps, "env_steps_per_s": n * steps / (ms * 1e-3),
           "ms_per_step": ms / steps, "views_ms_per_call": view_ms}
    print(json.dumps(rec), flush=True)
    return rec


def first_call(level, n):
    """Host-clock time of the first 160x120/16 call on a fresh batch against the next 50."""
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(LEVELS[level], n)
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
    env.close()
    rec = {"arm": "%s/first_call_160x120x16" % level, "first_ms": first, "later_ms": later}
    print(json.dumps(rec), flush=True)
    return rec


def main():
    import tempfile
    import numpy as np
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--episode-steps", type=int, default=20)
    ap.add_argument("--baseline-tree", metavar="DIR", help="built checkout of the revision to compare bench.py against")
    ap.add_argument("--bench-steps", type=int, default=200)
    ap.add_argument("--bench-warmup", type=int, default=20)
    ap.add_argument("--bench-only", action="store_true", help="skip part 1")
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    recs, firsts = [], []
    for _ in range(0 if args.bench_only else args.rounds):
        for level in LEVELS:
            for arm in ARMS:
                recs.append(run_arm(level, arm, args.envs, args.steps, args.warmup, args.episode_steps))
            firsts.append(first_call(level, args.envs))
    if recs:
        for level in LEVELS:
            for arm in ARMS:
                for key in ("env_steps_per_s", "views_ms_per_call")[:1 if arm == "step" else 2]:
                    w = np.array([r[key] for r in recs if r["arm"] == "%s/%s" % (level, arm)])
                    print(json.dumps({"summary": "%s/%s %s" % (level, arm, key), "median": float(np.median(w)),
                                      "min": float(w.min()), "max": float(w.max())}), flush=True)
            for k in ("first_ms", "later_ms"):
                w = np.array([r[k] for r in firsts if r["arm"].startswith(level)])
                print(json.dumps({"summary": "%s first_call %s" % (level, k), "median": float(np.median(w)),
                                  "min": float(w.min()), "max": float(w.max())}), flush=True)
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
