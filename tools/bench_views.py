"""Cost of designed-camera views (mwb_render_views, BatchedMiniWorld.render_views), measured on one GPU.

    python tools/bench_views.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3] [--episode-steps 20]
                                [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20] [--bench-only]

Part 1: 4096 envs of FourRooms and of PickupObjects, device-resident like bench.py's main arm, with episodes truncated
after `--episode-steps` steps (staggered) so that a twentieth of the envs reset in every step.  Four arms run
alternately for `--rounds` rounds:
  * step:  step only;
  * full:  step, then one view of every env from a row written by torch ops (1.5 m from the agent, facing it);
  * done:  step, then the ImageNav goal image: views only for the envs that just ended, every other row NaN (skipped);
  * pano:  step, then a four-heading panorama of every env (V = 4 views 90 degrees apart at the agent's position).
Each run prints one JSON line: env-steps/s from CUDA events, K1 / K2 time per launch from mwb_profile (the K2 average
covers the step's observation launch and the view launches), and the time of the render_views calls alone (CUDA
events around them) per call and per view.  After the arms, the time of an all-skipped call (every row NaN, one view)
is taken over 200 calls: the floor a skipped view costs.  A summary line per level and arm gives the median and the
spread (min, max) over the rounds.

Part 2 (with `--baseline-tree DIR`, a built checkout of another revision): `bench.py --gpus 1` (default config) and
`bench.py --gpus 1 --config 4` of DIR and of this tree, alternately, `--rounds` times each, then `--dump-outputs` of
both compared file by file (`--bench-only` runs part 2 alone).
The first line names the card and its power limit.  Nothing is written to either tree.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_level_changes import card  # noqa: E402
from bench_level_dr import run_bench, same_dumps, summary  # noqa: E402
from bench_reset_draws import short_level  # noqa: E402

LEVELS = {"fourrooms": "MiniWorld-FourRooms-v0", "pickup": "MiniWorld-PickupObjects-v0"}
ARMS = ("step", "full", "done", "pano")


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
    views = 4 if arm == "pano" else 1
    out = torch.zeros((views,) + env.obs_shape, dtype=torch.uint8, device=dev)
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

    def step(t, timed):
        _, _, te, tr, _ = env.step(acts[t])
        if arm == "step":
            return
        r = rows(te | tr)
        if timed:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
        env.render_views(r, out=out if arm == "pano" else out[0])
        if timed:
            b.record()
            ev.append((a, b))

    for t in range(warmup):
        step(t, False)
    torch.cuda.synchronize()
    env.engine.profile(True)
    env.engine.profile_read()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(warmup, warmup + steps):
        step(t, True)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    k1, k2, n1, n2 = env.engine.profile_read()
    env.engine.profile(False)
    view_ms = sum(a.elapsed_time(b) for a, b in ev) / max(len(ev), 1)
    rec = {"arm": "%s/%s" % (level, arm), "envs": n, "steps": steps, "env_steps_per_s": n * steps / (ms * 1e-3),
           "ms_per_step": ms / steps, "k1_ms_per_launch": k1 / max(n1, 1), "k2_ms_per_launch": k2 / max(n2, 1),
           "views_ms_per_call": view_ms, "views_ms_per_view": view_ms / views}
    if arm == "step":                      # the floor of a skipped view: one all-NaN view, 200 calls
        for _ in range(20):
            env.render_views(nan, out=out[0])
        torch.cuda.synchronize()
        e0.record()
        for _ in range(200):
            env.render_views(nan, out=out[0])
        e1.record()
        torch.cuda.synchronize()
        rec["all_skipped_ms_per_call"] = e0.elapsed_time(e1) / 200
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
    ap.add_argument("--bench-only", action="store_true", help="skip part 1")
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    recs = []
    for _ in range(0 if args.bench_only else args.rounds):
        for level in LEVELS:
            for arm in ARMS:
                recs.append(run_arm(level, arm, args.envs, args.steps, args.warmup, args.episode_steps))
    if recs:
        summary(recs)
    import numpy as np
    for level in LEVELS if recs else ():
        rs = [r for r in recs if r["arm"] == "%s/step" % level]
        v = np.array([r["all_skipped_ms_per_call"] for r in rs])
        for arm in ("full", "done", "pano"):
            w = np.array([r["views_ms_per_view"] for r in recs if r["arm"] == "%s/%s" % (level, arm)])
            print(json.dumps({"summary": "%s/%s views_ms_per_view" % (level, arm), "median": float(np.median(w)),
                              "min": float(w.min()), "max": float(w.max())}), flush=True)
        print(json.dumps({"summary": "%s all_skipped_ms_per_call" % level, "median": float(np.median(v)),
                          "min": float(v.min()), "max": float(v.max())}), flush=True)
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
