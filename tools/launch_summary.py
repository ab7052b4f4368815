"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list: the LAST complete iteration (between the
last two launches whose name matches --mark) grouped by kernel family.
    python tools/launch_summary.py launches.csv --mark head_loss"""
import csv, re, sys, collections

def family(name):
    n = name
    if "dwt::" in n:
        m = re.search(r"(cl_[a-z_]+?|tc_[a-z_]+?|small_[a-z_]+?|tiled_[a-z_]+?|vec_reduce|head_loss|mec|fwd_factor|bwd_coef|partial_reduce|augment_pair|maxpool_[a-z]+)(?:_3s2)?_kernel", n)
        return "dwt_b200: " + (m.group(1) if m else n[:40])
    low = n.lower()
    if "nchwtonhwc" in low or "nhwctonchw" in low: return "cuDNN layout conversion"
    if any(k in low for k in ("cudnn", "cutlass", "xmma", "sm90", "sm100", "sm80", "gemm", "conv", "wgrad", "dgrad", "implicit", "cublas", "gemv", "splitk")): return "cuDNN/cuBLAS conv + gemm"
    if "max_pool" in low or "maxpool" in low: return "ATen max-pool fwd/bwd"
    if "multi_tensor" in low or "foreach" in low: return "ATen foreach (optimizer / zero)"
    if "cholesky" in low or "potr" in low or "trsm" in low or "getr" in low or "inverse" in low or "lu_" in low or "magma" in low or "cusolver" in low: return "cuSOLVER/MAGMA factor + inverse"
    if "batch_norm" in low: return "ATen batch_norm"
    if "cat" in low and "kernel" in low: return "ATen cat"
    if "reduce" in low: return "ATen reduce"
    if "elementwise" in low or "vectorized" in low or "copy" in low or "fill" in low: return "ATen elementwise / copy"
    return "other: " + n[:60]

def main():
    path = sys.argv[1]
    mark = sys.argv[sys.argv.index("--mark") + 1] if "--mark" in sys.argv else None
    rows = []
    with open(path, newline="") as f:
        lines = [l for l in f if not l.startswith("==")]
    rd = csv.DictReader(lines)
    for r in rd:
        try:
            v = float(r["Metric Value"].replace(",", ""))
        except Exception:
            continue
        unit = r.get("Metric Unit", "ns")
        ns = v * {"ns": 1, "nsecond": 1, "us": 1e3, "usecond": 1e3, "ms": 1e6, "msecond": 1e6}.get(unit, 1)
        rows.append((r["Kernel Name"], ns))
    if mark:
        idx = [i for i, (n, _) in enumerate(rows) if mark in n]
        if len(idx) >= 2:
            rows = rows[idx[-2] + 1: idx[-1] + 1]
    tot = sum(ns for _, ns in rows)
    fam = collections.defaultdict(lambda: [0, 0.0])
    byname = collections.defaultdict(lambda: [0, 0.0])
    for n, ns in rows:
        fam[family(n)][0] += 1; fam[family(n)][1] += ns
        byname[n[:110]][0] += 1; byname[n[:110]][1] += ns
    print(f"total {tot/1e6:.3f} ms serialised, {len(rows)} launches\n")
    print("| kernel family | launches | summed us | share |\n|---|---|---|---|")
    for k, (c, ns) in sorted(fam.items(), key=lambda kv: -kv[1][1]):
        print(f"| {k} | {c} | {ns/1e3:.0f} | {100*ns/tot:.1f} % |")
    if "--names" in sys.argv:
        print("\n| kernel | launches | summed us | share |\n|---|---|---|---|")
        for k, (c, ns) in sorted(byname.items(), key=lambda kv: -kv[1][1])[:45]:
            print(f"| `{k}` | {c} | {ns/1e3:.0f} | {100*ns/tot:.1f} % |")

if __name__ == "__main__":
    main()
