"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel: count, total us, share."""
import csv, re, sys
from collections import defaultdict
rows = []
with open(sys.argv[1]) as fh:
    lines = [l for l in fh if not l.startswith("==")]
rd = csv.DictReader(lines)
agg = defaultdict(lambda: [0, 0.0])
total = 0.0
for r in rd:
    if r.get("Metric Name") != "gpu__time_duration.sum":
        continue
    name = r["Kernel Name"]
    v = float(r["Metric Value"].replace(",", ""))
    unit = r.get("Metric Unit", "ns")
    us = v / 1000.0 if unit in ("ns", "nsecond") else (v if unit in ("us", "usecond") else v * 1000.0)
    short = re.sub(r"\(.*$", "", name)[:90]
    agg[short][0] += 1
    agg[short][1] += us
    total += us
ours = ("fir4_band", "upfirdn2d_generic", "bias_act", "noise_bias_act", "bias_grad", "warp_", "mip_down", "flow_compose",
        "splat_", "demod_umma", "modulate_kernel", "wsq_kernel", "blur_nhwc", "channel_scale", "rowwise_", "nhwc_finish",
        "row_finish", "to_rgb_nhwc", "feature_distance", "distance_finish", "styled_tail", "tent_down", "fused_adam", "tv_loss",
        "nn_argmin", "lookup_splat", "warp_compose")
def is_ours(k):   # every kernel of libgg_b200 lives in namespace gg (the name list is kept for pre-namespace captures)
    return "gg::" in k or any(o in k for o in ours)


mine = sum(v[1] for k, v in agg.items() if is_ours(k))
print("total %.1f us over %d launches; hand-written kernels %.1f us (%.1f%%)" % (total, sum(v[0] for v in agg.values()), mine, 100 * mine / max(total, 1e-9)))
for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1])[: int(sys.argv[2]) if len(sys.argv) > 2 else 40]:
    tag = "*" if is_ours(k) else " "
    print("%s %6d %10.1f us %5.1f%%  %s" % (tag, n, us, 100 * us / total, k))
