"""Sum dram bytes of every conv_tc_kernel launch of ONE forward from an ncu csv (metrics pass):
  ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum -k regex:conv_tc_kernel -s 62 -c 62 \
      --csv --log-file conv_traffic.csv python tools/ncu_target.py v8n 32
  python tools/ncu_traffic.py conv_traffic.csv v8n 32 > conv_traffic.json"""
import csv
import json
import sys

rows = list(csv.DictReader(l for l in open(sys.argv[1]) if not l.startswith("==")))
tot = {"dram__bytes_read.sum": 0.0, "dram__bytes_write.sum": 0.0, "gpu__time_duration.sum": 0.0}
mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-9, "us": 1e-6, "usecond": 1e-6, "nsecond": 1e-9, "ms": 1e-3}
ids = set()
for r in rows:
    ids.add(r["ID"])
    tot[r["Metric Name"]] += float(r["Metric Value"].replace(",", "")) * mult.get(r["Metric Unit"], 1)
print(json.dumps({"model": sys.argv[2], "batch": int(sys.argv[3]), "launches": len(ids),
                  "dram_bytes_per_step": tot["dram__bytes_read.sum"] + tot["dram__bytes_write.sum"],
                  "dram_read": tot["dram__bytes_read.sum"], "dram_write": tot["dram__bytes_write.sum"],
                  "kernel_seconds_serialised": tot["gpu__time_duration.sum"],
                  "source": "ncu --metrics dram__bytes_{read,write}.sum over the conv_tc_kernel launches of one eager forward"}))
