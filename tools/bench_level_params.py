"""Cost of level params written while the batch runs (MWB_ARRAY_LEVEL_PARAMS, BatchedMiniWorld.set_level_param),
measured on one GPU.

    python tools/bench_level_params.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3]
                                       [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20]

Part 1: 4096 FourRooms envs with domain_rand on, device-resident like bench.py's main arm, three arms run
alternately for `--rounds` rounds:
  * never:  the params are never written;
  * every50: every 50 steps torch ops widen or narrow forward_step's and turn_step's ranges from the rewards of the
             last 50 steps (an automatic domain randomisation loop; no host sync);
  * every1: the same writes before every step.
Each run prints one JSON line (env-steps/s, K1 / K2 time per launch from mwb_profile); a summary line per arm gives
the median and the spread (min, max) over the rounds.

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

LEVEL = "MiniWorld-FourRooms-v0"
EVERY = {"never": 0, "every50": 50, "every1": 1}


def run_arm(arm, n, steps, warmup):
    import numpy as np
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    every = EVERY[arm]
    env = BatchedMiniWorld(LEVEL, n, domain_rand=True)
    env.reset(seed=1000)
    dev = torch.device("cuda", env.device)
    acts = torch.as_tensor(np.random.default_rng(12345).integers(0, env.single_action_space.n, size=(warmup + steps, n),
                                                                dtype=np.int32), device=dev)
    fs = torch.tensor([0.15, 0.12, 0.17], dtype=torch.float64, device=dev)
    ts = torch.tensor([15.0, 10.0, 20.0], dtype=torch.float64, device=dev)
    score = torch.zeros(n, dtype=torch.float64, device=dev)

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

    for t in range(warmup):
        step(t)
    torch.cuda.synchronize()
    env.engine.profile(True)
    env.engine.profile_read()
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
    rec = {"arm": arm, "envs": n, "steps": steps, "env_steps_per_s": n * steps / (ms * 1e-3), "ms_per_step": ms / steps,
           "k1_ms_per_launch": k1 / max(n1, 1), "k2_ms_per_launch": k2 / max(n2, 1)}
    p = env.get_level_params(0).params
    rec["forward_step_range_at_end"] = [p["forward_step"].min, p["forward_step"].max]
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
    ap.add_argument("--baseline-tree", metavar="DIR", help="built checkout of the revision to compare bench.py against")
    ap.add_argument("--bench-steps", type=int, default=200)
    ap.add_argument("--bench-warmup", type=int, default=20)
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    recs = []
    for _ in range(args.rounds):
        for arm in EVERY:
            recs.append(run_arm(arm, args.envs, args.steps, args.warmup))
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
