"""ncu_summary.py REPORT.ncu-rep [N_LINES] — text summary of an `ncu --set full --import-source on` capture: per launch the duration, DRAM
bytes, registers, occupancy limits, instruction counts, lanes per instruction, local / shared / global memory instructions, IPC, stall reasons, and the
top source lines by stall samples (needs -lineinfo).  Also prints one JSON line per launch with the DRAM traffic."""
import csv
import io
import json
import subprocess
import sys
import collections

rep = sys.argv[1]
N = int(sys.argv[2]) if len(sys.argv) > 2 else 25
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__waves_per_multiprocessor",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "sm__inst_executed.avg.per_cycle_active", "sass__inst_executed_local_loads", "sass__inst_executed_local_stores", "sass__inst_executed_shared_loads",
        "sass__inst_executed_global_loads", "smsp__cycles_active.avg", "sm__cycles_elapsed.max", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed"]


def num(s):
    try:
        return float(s.replace(",", ""))
    except Exception:
        return None


print("# %s" % rep)
for r in rows[2:]:
    d = dict(zip(hdr, r))
    u = dict(zip(hdr, units))
    print("== launch %s  %s" % (d.get("ID"), d.get("Kernel Name")))
    for w in WANT:
        if w in d:
            print("  %-58s %s %s" % (w, d[w], u[w]))
    stalls = sorted(((num(d[k]) or 0, k) for k in hdr if k.startswith("smsp__average_warps_issue_stalled_") and k.endswith("_per_issue_active.ratio")), reverse=True)
    for v, k in stalls[:8]:
        print("    stall %-40s %.2f warps / issue" % (k[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")], v))
    def to_bytes(key):
        v, un = num(d.get(key, "")), u.get(key, "")
        if v is None:
            return None
        return v * {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1}.get(un, 1)
    rd, wr = to_bytes("dram__bytes_read.sum"), to_bytes("dram__bytes_write.sum")
    print("  TRAFFIC_JSON " + json.dumps({"kernel": d.get("Kernel Name"), "dram_bytes_per_launch": (rd or 0) + (wr or 0), "read": rd, "write": wr,
                                          "duration_us": num(d.get("gpu__time_duration.sum", ""))}))

src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "cuda,sass"], capture_output=True, text=True).stdout
cur = kern = hdr2 = None
per = collections.OrderedDict()
for r in csv.reader(io.StringIO(src)):
    if len(r) == 2 and r[0] == "File Path":
        cur = r[1].split("/")[-1]; continue
    if len(r) == 2 and r[0] == "Function Name":
        kern = r[1]; per.setdefault(kern, []); continue
    if r and r[0] == "Line No":
        hdr2 = r; continue
    if not hdr2 or len(r) != len(hdr2) or not r[0].isdigit() or kern is None:
        continue
    ix = {n: i for i, n in enumerate(hdr2)}
    g = lambda n: int(r[ix[n]]) if r[ix[n]].lstrip("-").isdigit() else 0
    st = {n[6:]: g(n) for n in hdr2 if n.startswith("stall_") and "Not Issued" not in n}
    per[kern].append((cur, int(r[0]), r[1].strip()[:100], g("Instructions Executed"), g("# Samples"), g("Thread Instructions Executed"), st))
for kern, out in per.items():
    if not out:
        continue
    tot = sum(o[3] for o in out) or 1; ts = sum(o[4] for o in out) or 1; tt = sum(o[5] for o in out)
    print("\n== source view: %s\n  warp inst %d (all captured launches), thread inst %d, lanes / inst %.2f, samples %d" % (kern, tot, tt, tt / tot, ts))
    bf, sf, stc = collections.Counter(), collections.Counter(), collections.Counter()
    for o in out:
        bf[o[0]] += o[3]; sf[o[0]] += o[4]
        for k, v in o[6].items():
            stc[k] += v
    for k, v in bf.most_common(6):
        print("    %-28s inst %5.1f%%  samples %5.1f%%" % (k, 100 * v / tot, 100 * sf[k] / ts))
    print("    stall samples: " + ", ".join("%s %.1f%%" % (k, 100 * v / ts) for k, v in stc.most_common(8)))
    merged = collections.OrderedDict()
    for o in out:  # merge the per-launch duplicates of a line
        key = (o[0], o[1])
        m = merged.setdefault(key, [o[2], 0, 0, 0, collections.Counter()])
        m[1] += o[3]; m[2] += o[4]; m[3] += o[5]; m[4].update(o[6])
    for (f, l), m in sorted(merged.items(), key=lambda kv: -kv[1][2])[:N]:
        top = max(m[4].items(), key=lambda kv: kv[1])[0] if m[4] else "-"
        print("    %-22s %4d inst=%5.2f%% samp=%5.2f%% lanes=%4.1f %-10s %s" % (f, l, 100 * m[1] / tot, 100 * m[2] / ts, m[3] / max(m[1], 1), top, m[0]))
