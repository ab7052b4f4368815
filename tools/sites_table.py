"""bench.py --sites-out JSON -> a per-site markdown table.
    python tools/sites_table.py sites.json [bench_line.json] > sites.md"""
import json, sys

rows = json.load(open(sys.argv[1]))
bench = json.loads(open(sys.argv[2]).read().strip().splitlines()[-1]) if len(sys.argv) > 2 else {}
print("# Per-site kernel table, NHWC\n")
print("`python bench.py --sites-out ...` -- CUDA-event time of every launch of the hand-written kernels in the eager pass of the")
print("ResNet-50-DWT step (fused sites incl. the residual tail with the ReLU byte map, 64 images/domain, D = 3 domains per launch),")
print("grouped by kernel family and site geometry.  `frac` = algorithmic bytes / time / the HBM peak of the bench line")
print("(MEASURED_PEAKS.json, else the data sheet's 3350 GB/s).  The event brackets include the launch latency of every launch:")
print("small sites read low here.")
if bench:
    print(f"Step: {bench.get('eager_ms_per_step', 0):.2f} ms eager, {bench.get('ms_per_step', 0):.2f} ms as a CUDA-graph replay = "
          f"{bench.get('value', 0):.0f} images/s.\n")
print("| kernel | C | HW | gs | launches | us/launch | GB/s | frac | ms/step |")
print("|---|---|---|---|---|---|---|---|---|")
for r in rows:
    print(f"| {r['kernel']} | {r.get('C', '-')} | {r.get('HW', '-')} | {r.get('GS', '-')} | {r['launches']} | {r['us_per_launch']:.1f} | "
          f"{r['gbs']:.0f} | {r['frac_of_peak']:.2f} | {r['ms_per_step']:.3f} |")
