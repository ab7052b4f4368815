"""Condense an `ncu --set full` report into a few lines per kernel.
    ncu -i prof.ncu-rep --page raw --csv > raw.csv ; python tools/ncu_summary.py raw.csv [algorithmic-bytes-per-kernel ...]
Algorithmic bytes (optional, one per captured launch in order, e.g. 822083584 or 2E with E=...) add the traffic ratio."""
import csv, sys

KEEP = [("gpu__time_duration.sum", "duration"),
        ("dram__bytes_read.sum", "dram read"), ("dram__bytes_write.sum", "dram write"),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram throughput % of peak"),
        ("lts__t_sector_hit_rate.pct", "L2 hit rate %"),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe active %"),
        ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", "shared-memory wavefronts % of peak"),
        ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "LSU pipe %"),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots active %"),
        ("smsp__inst_executed.sum", "warp instructions"),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
        ("launch__registers_per_thread", "registers/thread"),
        ("launch__waves_per_multiprocessor", "waves/SM"),
        ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long-scoreboard /issue"),
        ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short-scoreboard /issue"),
        ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier /issue"),
        ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall wait /issue")]


def to_bytes(v, unit):
    mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}
    return float(v.replace(",", "")) * mult.get(unit, 1)


def main():
    rows = list(csv.reader(open(sys.argv[1])))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    alg = [float(a) for a in sys.argv[2:]]
    for n, r in enumerate(rows[2:]):
        name = r[idx["Kernel Name"]]
        grid = r[idx["Grid Size"]] if "Grid Size" in idx else ""
        block = r[idx["Block Size"]] if "Block Size" in idx else ""
        print("----")
        print(f"{'Kernel':44s} {name[:120]}")
        print(f"{'Grid / block':44s} {grid} / {block}")
        for key, label in KEEP:
            if key in idx and r[idx[key]] != "":
                print(f"{label:44s} {r[idx[key]]} {units[idx[key]]}")
        if "dram__bytes_read.sum" in idx:
            t = to_bytes(r[idx["dram__bytes_read.sum"]], units[idx["dram__bytes_read.sum"]]) + \
                to_bytes(r[idx["dram__bytes_write.sum"]], units[idx["dram__bytes_write.sum"]])
            line = f"{'-> DRAM traffic':44s} {t / 1e6:.1f} MB"
            if n < len(alg) and alg[n] > 0:
                line += f" / algorithmic {alg[n] / 1e6:.1f} MB = {t / alg[n]:.3f}"
            print(line)


if __name__ == "__main__":
    main()
