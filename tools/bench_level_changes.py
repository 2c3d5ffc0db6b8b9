"""Cost of level changes at resets (BatchedMiniWorld(dynamic_levels=True)), measured on one GPU.

    python tools/bench_level_changes.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3]
                                        [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20]

Part 1, a mix of levels (default 4096 envs over FourRooms, Hallway, OneRoom, PickupObjects, contiguous blocks),
device-resident like bench.py's main arm, three arms run alternately for `--rounds` rounds:
  * static:   level changes off;
  * idle:     level changes on, all weights zero (every reset keeps its level);
  * sampling: level changes on, weights replaced on the device every 50 steps by torch ops (no host sync).
Each run prints one JSON line: env-steps/s, K1 / K2 time per launch (CUDA events, mwb_profile) and, for the sampling
arm, how many envs changed level in the timed region.

Part 2 (with `--baseline-tree DIR`, a built checkout of another revision): `bench.py --gpus 1` of DIR and of this
tree, alternately in one session, `--rounds` times each, then `--dump-outputs` of both compared file by file.
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

DEFAULT_LEVELS = ["MiniWorld-FourRooms-v0", "MiniWorld-Hallway-v0", "MiniWorld-OneRoom-v0", "MiniWorld-PickupObjects-v0"]


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


def run_arm(arm, levels, n, steps, warmup):
    import numpy as np
    import torch
    from miniworld_b200.batched import BatchedMiniWorld
    env = BatchedMiniWorld(levels, n, dynamic_levels=arm != "static", level_seed=7)
    env.reset(seed=1000)
    dev = torch.device("cuda", env.device)
    acts = torch.as_tensor(np.random.default_rng(12345).integers(0, env.single_action_space.n, size=(warmup + steps, n),
                                                                dtype=np.int32), device=dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)

    def step(t):
        if arm == "sampling" and t % 50 == 0:
            env.level_weights.copy_(torch.rand(len(levels), device=dev, generator=gen))
        env.step(acts[t])

    for t in range(warmup):
        step(t)
    start = env.level_tensor.clone() if arm != "static" else None
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
    rec = {"arm": arm, "levels": levels, "envs": n, "steps": steps, "env_steps_per_s": n * steps / (ms * 1e-3),
           "ms_per_step": ms / steps, "k1_ms_per_launch": k1 / max(n1, 1), "k2_ms_per_launch": k2 / max(n2, 1)}
    if start is not None:
        rec["envs_whose_level_changed"] = int((env.level_tensor != start).sum())
    env.close()
    print(json.dumps(rec), flush=True)
    return rec


def run_bench(tree, label, args, dump=None):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps),
           "--warmup", str(args.bench_warmup), "--no-cpu"] + (["--dump-outputs", dump] if dump else [])
    out = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, check=True).stdout
    line = json.loads([s for s in out.splitlines() if s.startswith("{")][-1])
    rec = {"arm": "bench.py", "build": label, "env_steps_per_s": line["value"], "ms_per_step": line["ms_per_step"],
           "k1_ms_per_launch": line["roofline"]["k1_avg_ms"], "k2_ms_per_launch": line["roofline"]["kernel_avg_ms"]}
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--levels", nargs="+", default=DEFAULT_LEVELS)
    ap.add_argument("--baseline-tree", metavar="DIR", help="built checkout of the revision to compare bench.py against")
    ap.add_argument("--bench-steps", type=int, default=200)
    ap.add_argument("--bench-warmup", type=int, default=20)
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    for _ in range(args.rounds):
        for arm in ("static", "idle", "sampling"):
            run_arm(arm, list(args.levels), args.envs, args.steps, args.warmup)
    if not args.baseline_tree:
        return
    base = os.path.abspath(args.baseline_tree)
    for _ in range(args.rounds):
        run_bench(base, "baseline", args)
        run_bench(ROOT, "this tree", args)
    with tempfile.TemporaryDirectory() as tmp:
        a, b = os.path.join(tmp, "baseline"), os.path.join(tmp, "this")
        run_bench(base, "baseline", args, dump=a)
        run_bench(ROOT, "this tree", args, dump=b)
        names = sorted(os.listdir(a))
        same = names == sorted(os.listdir(b)) and all(filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False)
                                                      for f in names)
        print(json.dumps({"arm": "dump-outputs", "files": names, "byte_identical": same}), flush=True)


if __name__ == "__main__":
    main()
