"""Cost of Maze levels in a level table (BatchedMiniWorld(levels, per_env_worlds=True)), measured on one GPU.

    python tools/bench_maze_levels.py [--envs 4096] [--steps 200] [--warmup 20] [--rounds 3]
                                      [--baseline-tree DIR] [--bench-steps 200] [--bench-warmup 20]

Part 1, device-resident like bench.py's main arm, `--rounds` rounds of:
  * mix:         `--envs` envs over OneRoom, FourRooms, MazeS2, MazeS3 and Maze (8 x 8), contiguous blocks;
  * mix-no-maze: the same mix without Maze (what the 8 x 8 maze's HBM triangle lists cost the batch);
  * alone:       each level of the first mix alone, at its count in that mix.
Each run prints one JSON line: env-steps/s, K1 / K2 time per launch (CUDA events, mwb_profile) and the device memory
the batch holds per env (cudaMemGetInfo before and after construction).

Part 2 (with `--baseline-tree DIR`, a built checkout of another revision): `bench.py --gpus 1` of DIR and of this
tree, default config and `--config 4` (MazeS8), alternately, `--rounds` times each, then `--dump-outputs` of both
compared file by file.  The first line names the card and its power limit.  Nothing is written to either tree.
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

MIX = ["MiniWorld-OneRoom-v0", "MiniWorld-FourRooms-v0", "MiniWorld-MazeS2-v0", "MiniWorld-MazeS3-v0", "MiniWorld-Maze-v0"]


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
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    if isinstance(levels, str):
        env = BatchedMiniWorld(levels, n)
    else:
        env = BatchedMiniWorld(levels, n, per_env_worlds=True)
    env.reset(seed=1000)
    torch.cuda.synchronize()
    held = free0 - torch.cuda.mem_get_info()[0]
    dev = torch.device("cuda", env.device)
    acts = torch.as_tensor(np.random.default_rng(12345).integers(0, env.single_action_space.n, size=(warmup + steps, n),
                                                                dtype=np.int32), device=dev)
    for t in range(warmup):
        env.step(acts[t])
    torch.cuda.synchronize()
    env.engine.profile(True)
    env.engine.profile_read()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(warmup, warmup + steps):
        env.step(acts[t])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    k1, k2, n1, n2 = env.engine.profile_read()
    env.engine.profile(False)
    assert env.engine.overflow_count() == 0
    rec = {"arm": arm, "levels": levels, "envs": n, "steps": steps, "env_steps_per_s": n * steps / (ms * 1e-3),
           "ms_per_step": ms / steps, "k1_ms_per_launch": k1 / max(n1, 1), "k2_ms_per_launch": k2 / max(n2, 1),
           "device_bytes_per_env": held / n}
    env.close()
    print(json.dumps(rec), flush=True)
    return rec


def run_bench(tree, label, args, config=None, dump=None):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps),
           "--warmup", str(args.bench_warmup), "--no-cpu"] + (["--config", str(config)] if config is not None else []) + \
          (["--dump-outputs", dump] if dump else [])
    out = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, check=True).stdout
    line = json.loads([s for s in out.splitlines() if s.startswith("{")][-1])
    rec = {"arm": "bench.py", "config": config if config is not None else "default", "build": label,
           "env_steps_per_s": line["value"], "ms_per_step": line["ms_per_step"],
           "k1_ms_per_launch": line["roofline"]["k1_avg_ms"], "k2_ms_per_launch": line["roofline"]["kernel_avg_ms"]}
    print(json.dumps(rec), flush=True)
    return rec


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
    from miniworld_b200.batched import default_env_level
    import numpy as np
    counts = np.bincount(default_env_level(args.envs, len(MIX)), minlength=len(MIX))
    no_maze = MIX[:-1]
    for _ in range(args.rounds):
        run_arm("mix", MIX, args.envs, args.steps, args.warmup)
        run_arm("mix-no-maze", no_maze, int(counts[:-1].sum()), args.steps, args.warmup)
        for lv, c in zip(MIX, counts):
            run_arm("alone", lv, int(c), args.steps, args.warmup)
    if not args.baseline_tree:
        return
    base = os.path.abspath(args.baseline_tree)
    for config in (None, 4):
        for _ in range(args.rounds):
            run_bench(base, "baseline", args, config)
            run_bench(ROOT, "this tree", args, config)
        with tempfile.TemporaryDirectory() as tmp:
            a, b = os.path.join(tmp, "baseline"), os.path.join(tmp, "this")
            run_bench(base, "baseline", args, config, dump=a)
            run_bench(ROOT, "this tree", args, config, dump=b)
            names = sorted(os.listdir(a))
            same = names == sorted(os.listdir(b)) and all(
                filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False) for f in names)
            print(json.dumps({"arm": "dump-outputs", "config": config if config is not None else "default",
                              "files": names, "byte_identical": same}), flush=True)


if __name__ == "__main__":
    main()
