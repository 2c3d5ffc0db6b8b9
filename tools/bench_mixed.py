"""Cost of running several levels in one batch, measured on one GPU.

    python tools/bench_mixed.py [--envs 4096] [--steps 200] [--warmup 20] [--levels ID ID ...]

Arms (device-resident, like bench.py's main arm: actions, observations, rewards and flags stay in device memory):
  * mixed: one handle of `--envs` envs, the levels in contiguous near-equal blocks (BatchedMiniWorld's default);
  * alone: each level on its own handle with the same per-level env count.
Each arm prints one JSON line: env-steps/s, K1 / K2 time per launch (CUDA events, mwb_profile) and K2's block shape,
dynamic shared memory and resident blocks per SM (the `MWB_DEBUG` report of mwb_create).  The last line compares the
mixed step time with the sum of the levels' step times.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT_LEVELS = ["MiniWorld-FourRooms-v0", "MiniWorld-Hallway-v0", "MiniWorld-OneRoom-v0", "MiniWorld-PickupObjects-v0"]


def make_env(level, n, **kw):
    """BatchedMiniWorld with mwb_create's MWB_DEBUG line (K2 shared memory and occupancy) captured from stderr."""
    from miniworld_b200.batched import BatchedMiniWorld
    os.environ["MWB_DEBUG"] = "1"
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            env = BatchedMiniWorld(level, n, **kw)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["MWB_DEBUG"]
        f.seek(0)
        report = [line.strip() for line in f if line.startswith("[mwb] K2")]
    return env, (report[-1] if report else "")


def run_arm(name, level, n, steps, warmup, **kw):
    import numpy as np
    import torch
    env, k2 = make_env(level, n, **kw)
    env.reset(seed=1000)
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
    k1, k2_ms, n1, n2 = env.engine.profile_read()
    env.engine.profile(False)
    assert env.engine.overflow_count() == 0
    rec = {"arm": name, "levels": level if isinstance(level, list) else [level], "envs": n, "steps": steps,
           "env_steps_per_s": n * steps / (ms * 1e-3), "ms_per_step": ms / steps,
           "k1_ms_per_launch": k1 / max(n1, 1), "k2_ms_per_launch": k2_ms / max(n2, 1), "k2_launches_per_step": n2 / steps,
           "tri_cap": 2 * (env.engine.cfg.max_quads + 6 * env.engine.cfg.max_ents) + 2, "k2_report": k2}
    env.close()
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--levels", nargs="+", default=DEFAULT_LEVELS)
    args = ap.parse_args()
    import torch
    print(json.dumps({"gpu": torch.cuda.get_device_name(0)}), flush=True)
    mixed = run_arm("mixed", list(args.levels), args.envs, args.steps, args.warmup)
    per = args.envs // len(args.levels)
    alone = [run_arm("alone", lv, per, args.steps, args.warmup) for lv in args.levels]
    parts = sum(a["ms_per_step"] for a in alone)
    print(json.dumps({"arm": "summary", "mixed_ms_per_step": mixed["ms_per_step"], "sum_of_levels_ms_per_step": parts,
                      "mixed_over_sum": mixed["ms_per_step"] / parts}), flush=True)


if __name__ == "__main__":
    main()
