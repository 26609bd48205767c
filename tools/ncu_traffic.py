"""Mean DRAM traffic per launch of one kernel family in an .ncu-rep -> profiles/<name>.json (read by bench.py for
roofline.traffic).  python tools/ncu_traffic.py gpurun_out/prof_gemm.ncu-rep gemm_tile_kernel profiles/r1_gemm_traffic.json"""
import csv, json, subprocess, sys

UNIT = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
rep, pattern, dst = sys.argv[1:4]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr, units = rows[0], rows[1]
ir, iw, it = (hdr.index(k) for k in ("dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__time_duration.sum"))
tot, n, us = 0.0, 0, 0.0
for row in rows[2:]:
    if pattern not in row[hdr.index("Kernel Name")]:
        continue
    tot += float(row[ir]) * UNIT[units[ir]] + float(row[iw]) * UNIT[units[iw]]
    us += float(row[it]) * {"us": 1.0, "ns": 1e-3, "ms": 1e3}.get(units[it], 1.0)
    n += 1
json.dump({"kernel": pattern, "launches_captured": n, "dram_bytes_per_launch": tot / n, "mean_us_under_ncu": us / n,
           "source": rep.split("/")[-1], "note": "ncu --set full, cold caches (ncu flushes L2 between replays): every "
           "operand is fetched from DRAM once; in the running loop part of the weights and activations stays in the 50 MB L2"},
          open(dst, "w"), indent=1)
print(open(dst).read())
