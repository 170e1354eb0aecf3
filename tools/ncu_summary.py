"""Key metrics of ncu reports (read here, without a GPU): python tools/ncu_summary.py *.ncu-rep"""
import csv
import io
import subprocess
import sys

WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor.sum", "sm__pipe_tensor_op_hmma_cycles_active.avg.pct_of_peak_sustained_active", "l1tex__t_bytes.sum", "lts__t_bytes.sum",
        "sm__inst_executed.sum", "smsp__cycles_active.avg", "sm__ops_path_tensor_op_utchmma_src_fp16_dst_fp32_sparsity_off.avg.pct_of_peak_sustained_elapsed",
        "sm__ops_path_tensor_src_fp16_dst_fp32.avg.pct_of_peak_sustained_elapsed", "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"]

for path in sys.argv[1:]:
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    if len(rows) < 3:
        print(path, "no data"); continue
    hdr, units = rows[0], rows[1]
    for vals in rows[2:]:
        d = dict(zip(hdr, vals))
        u = dict(zip(hdr, units))
        print(f"== {path}: {d.get('Kernel Name', '?')[:90]}")
        for k in hdr:
            if k in WANT:
                print(f"   {k:75s} {d[k]:>16s} {u[k]}")
