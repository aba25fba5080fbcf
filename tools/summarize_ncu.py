"""Condenses an .ncu-rep capture (ncu --set full) into the few numbers the roofline discussion needs.
    python tools/summarize_ncu.py prof.ncu-rep > prof_summary.txt
Runs here (no GPU needed): it only reads the report with `ncu -i`."""
import csv
import io
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__registers_per_thread", "regs/thread"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem/block"),
    ("launch__waves_per_multiprocessor", "waves/SM"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput % of peak"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 throughput % of peak"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput % of peak"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe % active"),
    ("sm__inst_executed_pipe_tensor.sum", "tensor instructions"),
    ("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "FMA pipe % active"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots % busy"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smem bank conflicts"),
]


def main(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    print("# %s" % path)
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")]
        print("\n## %s" % name[:150])
        for key, label in KEYS:
            if key in hdr:
                i = hdr.index(key)
                print("  %-34s %s %s" % (label, r[i], units[i]))
        # any tensor-pipe metric present
        for i, h in enumerate(hdr):
            if "pipe_tensor" in h and "pct" in h and r[i] not in ("", "0", "n/a") and h not in dict(KEYS):
                print("  %-34s %s %s" % (h[:34], r[i], units[i]))


if __name__ == "__main__":
    main(sys.argv[1])
