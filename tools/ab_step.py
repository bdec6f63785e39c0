"""A/B of the training step between two source trees on ONE card, in one call:

    python tools/ab_step.py --parent build/parent [--runs 3] [--out DIR]

1. `bench.py --gpus 1 --steps 20 --warmup 5 --dump-outputs` alternately in the parent tree and in this one, `--runs` times
   each: fp32 and bf16 ms_per_step of every run, their spread, and the roofline kernel's achieved bandwidth;
2. the `--dump-outputs` directories of the two trees (fp32, and bf16 from one extra `--dtype bf16` run per tree) compared
   byte for byte;
3. one eager step per tree and storage type under torch.profiler (CUDA activities), in a process of its own: time per
   kernel name.
The card's name and power limit are read alongside (a query; nothing is set).  `--parent` is a built export of the commit
to compare against (`git archive <commit> | tar -x -C build/parent`, then `python -m gangealing_b200.build` there)."""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:
        return "unknown (%r)" % (exc,)


def bench(tree, dump, extra=()):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "20", "--warmup", "5", "--no-cpu-baseline", "--dump-outputs", dump]
    res = subprocess.run(cmd + list(extra), cwd=tree, capture_output=True, text=True)
    lines = [l for l in res.stdout.splitlines() if l.startswith("{")]
    if res.returncode != 0 or not lines:
        raise RuntimeError("bench.py failed in %s:\n%s" % (tree, res.stderr[-3000:]))
    return json.loads(lines[-1])


def profile_child(dtype, batch):
    """One eager training step of the tree in the working directory under torch.profiler -> JSON {kernel name: [us, calls]}."""
    sys.path.insert(0, os.getcwd())
    import torch
    from torch.profiler import ProfilerActivity, profile
    from gangealing_b200.training import TrainConfig, Trainer
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    tr = Trainer(TrainConfig(batch=batch, dtype=dtype), "cuda")
    for _ in range(4):
        tr.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tr.step()
        torch.cuda.synchronize()
    table = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            us, n = table.get(ev.name, (0.0, 0))
            table[ev.name] = (us + ev.device_time_total, n + 1)
    print("PROFILE " + json.dumps(table))


def profile_tree(tree, dtype, batch):
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "--profile-child", dtype, "--batch", str(batch)], cwd=tree,
                         capture_output=True, text=True)
    lines = [l for l in res.stdout.splitlines() if l.startswith("PROFILE ")]
    if res.returncode != 0 or not lines:
        raise RuntimeError("profile failed in %s:\n%s" % (tree, res.stderr[-3000:]))
    return json.loads(lines[-1][8:])


def short(name):
    name = name.replace("gg::(anonymous namespace)::", "").replace("void ", "")
    return name if len(name) <= 86 else name[:83] + "..."


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=os.path.join(HERE, "build", "parent"))
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--out", default=None, help="where the output dumps go (default: a temporary directory)")
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--profile-child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.profile_child:
        return profile_child(args.profile_child, args.batch)
    trees = {"parent": os.path.abspath(args.parent), "change": HERE}
    out = args.out or tempfile.mkdtemp(prefix="ab_step_")
    print("card: %s  (name, power limit, max SM clock)" % card(), flush=True)
    ms = {(t, d): [] for t in trees for d in ("f32", "bf16")}
    roof = {(t, d): [] for t in trees for d in ("f32", "bf16")}
    for r in range(args.runs):
        for t, tree in trees.items():
            line = bench(tree, os.path.join(out, t + "_f32"))
            ms[t, "f32"].append(line["ms_per_step"])
            ms[t, "bf16"].append(line["config3_bf16"]["ms_per_step"])
            roof[t, "f32"].append(line["roofline"]["achieved"])
            roof[t, "bf16"].append(line["config3_bf16"]["roofline"]["achieved"])
            print("run %d %-6s fp32 %.3f ms  bf16 %.3f ms   roofline kernel %.0f / %.0f GB/s" % (
                r, t, ms[t, "f32"][-1], ms[t, "bf16"][-1], roof[t, "f32"][-1], roof[t, "bf16"][-1]), flush=True)
    for t, tree in trees.items():
        bench(tree, os.path.join(out, t + "_bf16"), ["--dtype", "bf16", "--no-extra"])
    for d in ("f32", "bf16"):
        a, b = ms["parent", d], ms["change", d]
        ma, mb = sum(a) / len(a), sum(b) / len(b)
        print("%-4s ms_per_step  parent %.3f (%.3f..%.3f)  change %.3f (%.3f..%.3f)  change/parent %.4f  (%+.2f %%)" % (
            d, ma, min(a), max(a), mb, min(b), max(b), mb / ma, 100 * (mb / ma - 1)))
    same = True
    for d in ("f32", "bf16"):
        pa, pb = os.path.join(out, "parent_" + d), os.path.join(out, "change_" + d)
        names = sorted(set(os.listdir(pa)) | set(os.listdir(pb)))
        _, mismatch, errors = filecmp.cmpfiles(pa, pb, names, shallow=False)
        same = same and not mismatch and not errors
        print("outputs %-4s: %d files, %s" % (d, len(names), "byte-identical" if not mismatch and not errors
                                              else "DIFFER: %s" % (mismatch + errors)))
    if not args.no_profile:
        for d in ("f32", "bf16"):
            tabs = {t: profile_tree(tree, d, args.batch) for t, tree in trees.items()}
            names = sorted(set(tabs["parent"]) | set(tabs["change"]),
                           key=lambda k: -max(tabs["parent"].get(k, (0, 0))[0], tabs["change"].get(k, (0, 0))[0]))
            tot = {t: sum(v[0] for v in tabs[t].values()) for t in trees}
            print("\nper-kernel time of one eager %s step (us, launches): parent total %.0f us, change total %.0f us" % (
                d, tot["parent"], tot["change"]))
            print("%-86s %12s %5s %12s %5s" % ("kernel", "parent us", "n", "change us", "n"))
            for k in names[:40]:
                p, c = tabs["parent"].get(k, (0.0, 0)), tabs["change"].get(k, (0.0, 0))
                print("%-86s %12.0f %5d %12.0f %5d" % (short(k), p[0], p[1], c[0], c[1]))
            rest = names[40:]
            print("%-86s %12.0f %5d %12.0f %5d" % ("(%d more)" % len(rest), sum(tabs["parent"].get(k, (0, 0))[0] for k in rest), 0,
                                                   sum(tabs["change"].get(k, (0, 0))[0] for k in rest), 0))
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    main()
