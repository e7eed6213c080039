"""Run right after an `ncu --set full` capture: turns the (large) .ncu-rep into small text summaries -- the key metrics of every captured kernel (markdown table) and the executed-instruction
histogram by opcode with stall samples (from the source page).   python bench_micro/ncu_summarise.py <rep> <out_prefix>"""
import csv, io, subprocess, sys
from collections import Counter

rep, out = sys.argv[1], sys.argv[2]
KEYS = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
        "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_subpipe_imma_cycles_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__warps_eligible.avg.per_cycle_active",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_dispatch_stall_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio", "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "smsp__inst_executed.sum", "sass__inst_executed_local_loads", "sass__inst_executed_local_stores",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "lts__t_bytes.sum", "sm__cycles_elapsed.max"]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
name_col = hdr.index("Kernel Name") if "Kernel Name" in hdr else None
with open(out + "_metrics.md", "w") as f:
    f.write("# ncu --set full --clock-control none: key metrics per captured kernel (%s)\n\n" % rep)
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        f.write("## %s\n\n| metric | value | unit |\n|---|---|---|\n" % (d.get("Kernel Name", "?")[:160]))
        for k in KEYS:
            if k in d:
                f.write("| %s | %s | %s |\n" % (k, d[k], units[hdr.index(k)]))
        f.write("\n")
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
kernel, hist, samples, total = None, Counter(), Counter(), 0
reasons, by_op_reason, stall_cols = Counter(), {}, []
with open(out + "_opcodes.md", "w") as f:
    def flush():
        if kernel is None or not hist:
            return
        f.write("## %s\n\ntotal stall samples %d\n\n| opcode | warp instructions executed | stall samples | share |\n|---|---|---|---|\n" % (kernel[:160], total))
        for op, n in hist.most_common(28):
            f.write("| %s | %d | %d | %.1f %% |\n" % (op, n, samples[op], 100.0 * samples[op] / max(1, total)))
        f.write("\n")
        if reasons:
            tot = max(1, sum(reasons.values()))
            f.write("warp-state samples by reason (all instructions): " + ", ".join("%s %.1f %%" % (k, 100.0 * v / tot) for k, v in reasons.most_common(12)) + "\n\n")
            f.write("| opcode | top warp states while this opcode is next to issue |\n|---|---|\n")
            for op, _ in samples.most_common(10):
                c = by_op_reason.get(op, Counter()); t = max(1, sum(c.values()))
                f.write("| %s | %s |\n" % (op, ", ".join("%s %.0f %%" % (k, 100.0 * v / t) for k, v in c.most_common(4))))
            f.write("\n")
    cols = None
    for r in csv.reader(io.StringIO(src)):
        if r and r[0] == "Kernel Name":
            flush()
            kernel, hist, samples, total, cols = r[1], Counter(), Counter(), 0, None
            reasons, by_op_reason = Counter(), {}
            continue
        if r and r[0] == "Address":
            cols = (r.index("Source"), r.index("# Samples"), r.index("Instructions Executed"))
            stall_cols = [(i, h) for i, h in enumerate(r) if h.startswith("stall_") and "Not Issued" not in h]
            continue
        if cols and len(r) > max(cols):
            parts = r[cols[0]].split()
            if not parts:
                continue
            op = parts[1] if parts[0].startswith("@") and len(parts) > 1 else parts[0]
            try:
                s, n = int(r[cols[1]] or 0), int(r[cols[2]] or 0)
            except ValueError:
                continue
            hist[op] += n; samples[op] += s; total += s
            for i, h in stall_cols:
                try:
                    v = int(r[i] or 0)
                except (ValueError, IndexError):
                    continue
                if v:
                    reasons[h] += v
                    by_op_reason.setdefault(op, Counter())[h] += v
    flush()
print("wrote", out + "_metrics.md", out + "_opcodes.md")
