"""Cost of env params (mwb_enable_env_params, BatchedMiniWorld(env_params=True)), measured on one GPU.

    python tools/bench_env_params.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3] [--episode-steps 20]
                                      [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20]

Part 1: 4096 envs of FourRooms and of PickupObjects with domain randomisation, device-resident like bench.py's main
arm, with episodes truncated after `--episode-steps` steps so that a twentieth of the envs reset in every step.  Three
arms run alternately for `--rounds` rounds:
  * off:  env params off;
  * idle: env params on, never written: every reset writes a NaN row, every step merges nothing;
  * adr:  env params on, and after every step the README's ADR loop in torch ops gives every done env a design (with
          probability 0.5 one random element pinned at its level's lower or upper bound, otherwise an all-NaN row),
          with no host sync.
Each run prints one JSON line (env-steps/s from CUDA events, K1 / K2 time per launch from mwb_profile, and the device
memory the batch holds per env, from cudaMemGetInfo around its construction); a summary line per level and arm gives
the median and the spread (min, max) over the rounds.  Then the same rounds run again under torch.profiler (CUDA
activity only, no timing of their own) for K1's device time per launch.

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


def adr_update(env, done, gen):
    """The README ADR step: each done env pins one random element at its level's current lower or upper bound with
    probability 0.5, otherwise gets an all-NaN row; both set the pending flag."""
    import torch
    from miniworld_b200.engine import ENV_PARAM_ELEMS, PARAMS_COLUMN
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

LEVELS = {"fourrooms": "MiniWorld-FourRooms-v0", "pickup": "MiniWorld-PickupObjects-v0"}
ARMS = ("off", "idle", "adr")


def short_level(name, steps):
    """The level truncated after `steps` steps: frequent resets."""
    from miniworld_b200.envs import LEVELS as REGISTRY
    base = REGISTRY[name]

    def __init__(self, **kw):
        base.__init__(self, **kw)
        self.max_episode_steps = steps
    return type("Short" + base.__name__, (base,), {"__init__": __init__})


def run_arm(level, arm, n, steps, warmup, episode_steps, profile=False):
    import numpy as np
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    dev = torch.device("cuda", 0)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    env = BatchedMiniWorld(short_level(LEVELS[level], episode_steps), n, domain_rand=True, env_params=arm != "off")
    env.reset(seed=1000)
    torch.cuda.synchronize()
    bytes_per_env = (free0 - torch.cuda.mem_get_info(dev)[0]) / n
    acts = torch.as_tensor(np.random.default_rng(12345).integers(0, 3, size=(warmup + steps, n), dtype=np.int32), device=dev)
    # staggered starts, so that the resets spread over the steps instead of all falling into one
    stagger = torch.as_tensor(env.engine.state_array("step_count"), device=dev)
    stagger.copy_(torch.arange(n, device=dev, dtype=torch.int32) % episode_steps)
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)

    def step(t):
        _, _, te, tr, _ = env.step(acts[t])
        if arm == "adr":
            adr_update(env, te | tr, gen)

    for t in range(warmup):
        step(t)
    torch.cuda.synchronize()
    env.engine.profile(not profile)
    env.engine.profile_read()
    done0 = int(env.get_state()["episodes_done"][0])
    if profile:          # a run of its own: K1's device time per launch from torch.profiler's CUDA activity
        from torch.profiler import ProfilerActivity, profile as torch_profile
        with torch_profile(activities=[ProfilerActivity.CUDA]) as prof:
            for t in range(warmup, warmup + steps):
                step(t)
            torch.cuda.synchronize()
        k1 = [e for e in prof.events() if "step_kernel" in e.name]
        us = sum(e.device_time for e in k1) / max(len(k1), 1)
        env.engine.profile(False)
        env.close()
        rec = {"arm": "%s/%s" % (level, arm), "profiler": "torch", "k1_launches": len(k1), "k1_us_per_launch": us}
        print(json.dumps(rec), flush=True)
        return rec
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
           "device_bytes_per_env": bytes_per_env}
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
    recs = []
    for _ in range(args.rounds):
        for level in LEVELS:
            for arm in ARMS:
                recs.append(run_arm(level, arm, args.envs, args.steps, args.warmup, args.episode_steps, profile=True))
    for level in LEVELS:
        for arm in ARMS:
            v = sorted(r["k1_us_per_launch"] for r in recs if r["arm"] == "%s/%s" % (level, arm))
            print(json.dumps({"summary": "%s/%s" % (level, arm), "profiler": "torch", "k1_us_per_launch":
                              {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}}), flush=True)
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
