"""A/B of this tree against a baseline checkout on the C4 benchmark, in one GPU session.

    git archive <base> | tar -x -C build/ab_base      # once, then build both trees
    python tools/ab_bench.py --base build/ab_base --out build/ab_out [--ops 4,5,7,8,26] [--r50]

Prints the card, power limit and max SM clock; runs `bench.py` of the baseline and of this tree alternately (three runs
each, `--steps 30 --warmup 5 --no-cpu-baseline --sustained-seconds 0 --dump-outputs`); compares the dumps of the two arms
byte for byte; forwards the bench frames through both builds with the first block's pooled tensor requested (fused block
forced on) and compares those byte for byte; runs one more bench per arm with `BENCH_VERBOSE=1 SB_DEBUG=1` and prints the
per-op times and the autotune lines of the ops named by --ops (and the first block's); with --r50, one
`tools/bench_configs.py r50` run per arm.  A summary goes to <out>/summary.json."""
import argparse
import filecmp
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH_ARGS = ["--gpus", "1", "--steps", "30", "--warmup", "5", "--no-cpu-baseline", "--sustained-seconds", "0"]


def pooled(root, out_path):
    """Forward make_frames(8) through the C4 model of the tree at `root`; save the first block's pooled tensor."""
    sys.path.insert(0, root)
    os.environ["SB_FORCE_CONV01"] = "1"
    import numpy as np
    import bench
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn import oplist as ol
    from sleap_b200.nn.model import DeviceModel
    from sleap_b200._lib import ptr
    from ctypes import c_void_p
    spec = bench.c4_spec()
    cm = A.compile_model(spec, 1)
    m = DeviceModel(spec, A.make_synthetic_weights(cm, bench.SEED), input_channels=1, precision=0)
    frames = bench.make_frames(8)
    B, H, W, _ = frames.shape
    ops = cm.ops_array()
    pb = next(int(r[18]) for r in ops if r[0] == ol.CONV and r[18] >= 0)
    br = next(r for r in ops if r[0] == ol.BUFFER and r[1] == pb)
    out = np.zeros((B, H // int(br[2]), W // int(br[2]), int(br[3])), np.float32)
    m.configure(B, H, W, 1)
    ids = np.asarray([pb], np.int32)
    m.handle.call("sb_model_forward", m.model_id, ptr(frames), 1, B, 1, ptr(ids), (c_void_p * 1)(out.ctypes.data))
    np.save(out_path, out)


def run_bench(root, dump, env_extra=None):
    env = dict(os.environ, **(env_extra or {}))
    r = subprocess.run([sys.executable, "bench.py"] + BENCH_ARGS + ["--dump-outputs", dump], cwd=root, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        sys.stderr.write(r.stdout[-4000:] + r.stderr[-4000:])
        raise SystemExit(f"bench failed in {root} (exit {r.returncode})")
    return json.loads(lines[-1]), r.stderr


def same_tree(a, b):
    cmp = filecmp.dircmp(a, b)
    bad = cmp.left_only + cmp.right_only + cmp.funny_files
    _, mismatch, errors = filecmp.cmpfiles(a, b, cmp.common_files, shallow=False)
    bad += mismatch + errors
    for d in cmp.common_dirs:
        bad += [os.path.join(d, x) for x in same_tree(os.path.join(a, d), os.path.join(b, d))]
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default=os.path.join(HERE, "build", "ab_base"))
    ap.add_argument("--out", default=os.path.join(HERE, "build", "ab_out"))
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--ops", default="1", help="comma-separated op indices whose per-op times and autotune lines are printed")
    ap.add_argument("--r50", action="store_true", help="also run tools/bench_configs.py r50 once per arm")
    ap.add_argument("--pooled", metavar="NPY", help=argparse.SUPPRESS)
    ap.add_argument("--root", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.pooled:
        return pooled(args.root, args.pooled)
    base, new, out = os.path.abspath(args.base), HERE, os.path.abspath(args.out)
    os.makedirs(out, exist_ok=True)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         stdout=subprocess.PIPE, text=True).stdout, flush=True)
    arms = {"base": base, "new": new}
    res = {a: [] for a in arms}
    for i in range(args.runs):
        for a, root in arms.items():
            j, _ = run_bench(root, os.path.join(out, f"dump_{a}_{i}"))
            res[a].append(j)
            print(a, i, json.dumps({"value": j["value"], "e2e": j["e2e"]["value"],
                                    "kernel_ms_per_step": j["roofline"]["kernel_ms_per_step"],
                                    "precision2": j.get("strict_tensor_core", {}).get("value")}), flush=True)
    diff = same_tree(os.path.join(out, "dump_base_0"), os.path.join(out, "dump_new_0"))
    print("dump files that differ:", diff or "none", flush=True)
    import numpy as np
    for a, root in arms.items():
        subprocess.run([sys.executable, os.path.join(new, "tools", "ab_bench.py"), "--root", root, "--pooled",
                        os.path.join(out, f"pooled_{a}.npy")], cwd=root, check=True)
    pb, pn = np.load(os.path.join(out, "pooled_base.npy")), np.load(os.path.join(out, "pooled_new.npy"))
    pooled_same = pb.shape == pn.shape and pb.tobytes() == pn.tobytes()
    print("pooled tensor", pb.shape, "byte-identical:", pooled_same, flush=True)
    verbose = {}
    for a, root in arms.items():
        j, err = run_bench(root, os.path.join(out, f"dump_{a}_verbose"), {"BENCH_VERBOSE": "1", "SB_DEBUG": "1"})
        with open(os.path.join(out, f"verbose_{a}.log"), "w") as f:
            f.write(err)
        verbose[a] = j
        ops = [int(o) for o in args.ops.split(",")]
        keep = tuple(f"[op {o:2d}]" for o in ops) + tuple(f"[sb_conv_tc] op {o} launch" for o in ops)
        print(f"--- {a} autotune / per-op lines ---")
        print("\n".join(l for l in err.splitlines() if l.startswith(keep) or "first block" in l), flush=True)
    r50 = {}
    for a, root in arms.items() if args.r50 else ():
        r = subprocess.run([sys.executable, os.path.join("tools", "bench_configs.py"), "r50"], cwd=root, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
        lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
        r50[a] = json.loads(lines[-1]) if lines else None
        print(a, "r50", lines[-1] if lines else r.stdout[-2000:] + r.stderr[-2000:], flush=True)
    with open(os.path.join(out, "summary.json"), "w") as f:
        json.dump(dict(runs=res, verbose=verbose, dump_diff=diff, pooled_identical=pooled_same, r50=r50), f, indent=1)
    for a in arms:
        for key, get in (("value", lambda r: r["value"]), ("precision 2", lambda r: r["strict_tensor_core"]["value"])):
            v = sorted(get(r) for r in res[a])
            print(a, key, "median", v[len(v) // 2], "range", v[0], v[-1])


if __name__ == "__main__":
    main()
