"""Cost of per-level domain randomisation (mwb_level.domain_rand), measured on one GPU.

    python tools/bench_level_dr.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3]
                                   [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20]

Part 1: 4096 FourRooms envs as a table of three rows, device-resident like bench.py's main arm, three arms run
alternately for `--rounds` rounds:
  * off:    three rows, all with domain_rand off;
  * on:     three rows, all with domain_rand on;
  * ladder: off / on with ranges narrowed to a quarter / on, envs starting on row 0 and moved by weights that torch
            ops rewrite on the device every 50 steps (level changes on, no host sync).
Each run prints one JSON line (env-steps/s, K1 / K2 time per launch from mwb_profile); a summary line per arm gives
the median and the spread (min, max) over the rounds.

Part 2 (with `--baseline-tree DIR`, a built checkout of another revision): `bench.py --gpus 1` (default config) and
`bench.py --gpus 1 --config 4` (MazeS8 with randomisation) of DIR and of this tree, alternately, `--rounds` times
each, then `--dump-outputs` of both compared file by file for both configs.
The first line names the card and its power limit.  Nothing is written to either tree (dumps go to a temporary
directory).
"""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_level_changes import card  # noqa: E402

LEVEL = "MiniWorld-FourRooms-v0"


def narrowed_params(frac=0.25):
    """DEFAULT_PARAMS with every range shrunk to `frac` of its width around the default."""
    import numpy as np
    from miniworld_b200.params import DEFAULT_PARAMS
    p = DEFAULT_PARAMS.copy()
    for name, q in DEFAULT_PARAMS.params.items():
        if isinstance(q.default, np.ndarray):
            lo, hi = q.default - frac * (q.default - q.min), q.default + frac * (q.max - q.default)
        else:
            lo, hi = float(q.default - frac * (q.default - q.min)), float(q.default + frac * (q.max - q.default))
        p.set(name, q.default, lo, hi, q.type)
    return p


def rows_of(arm):
    if arm == "off":
        return [{"domain_rand": False}] * 3
    if arm == "on":
        return [{"domain_rand": True}] * 3
    return [{"domain_rand": False}, {"domain_rand": True, "params": narrowed_params()}, {"domain_rand": True}]


def run_arm(arm, n, steps, warmup):
    import numpy as np
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    ladder = arm == "ladder"
    kw = dict(env_level=np.zeros(n, np.int32), dynamic_levels=True, level_seed=7) if ladder else {}
    env = BatchedMiniWorld([LEVEL] * 3, n, level_kwargs=rows_of(arm), **kw)
    env.reset(seed=1000)
    dev = torch.device("cuda", env.device)
    acts = torch.as_tensor(np.random.default_rng(12345).integers(0, env.single_action_space.n, size=(warmup + steps, n),
                                                                dtype=np.int32), device=dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)

    def step(t):
        if ladder and t % 50 == 0:
            env.level_weights.copy_(torch.rand(3, device=dev, generator=gen))
        env.step(acts[t])

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
    if ladder:
        rec["envs_per_row_at_end"] = np.bincount(env.env_level, minlength=3).tolist()
    env.close()
    print(json.dumps(rec), flush=True)
    return rec


def summary(recs, label_key="arm"):
    import numpy as np
    groups = {}
    for r in recs:
        groups.setdefault((r[label_key], r.get("build"), r.get("config")), []).append(r)
    for (arm, build, config), rs in groups.items():
        out = {"summary": arm, "runs": len(rs)}
        if build:
            out.update(build=build, config=config)
        for key in ("env_steps_per_s", "k1_ms_per_launch", "k2_ms_per_launch"):
            v = np.array([r[key] for r in rs])
            out[key] = {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}
        print(json.dumps(out), flush=True)


def run_bench(tree, label, args, config=None, dump=None):
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


def same_dumps(a, b):
    names = sorted(os.listdir(a))
    return names, names == sorted(os.listdir(b)) and all(
        filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False) for f in names)


def main():
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
        for arm in ("off", "on", "ladder"):
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
