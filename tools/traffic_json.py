"""Write traffic entries from `ncu --page raw --csv` exports of the dominant kernel (tools/ncu_capture.sh):
    python tools/traffic_json.py profiles/traffic.json tet1m=ncu_out/x_raw.csv cart128=ncu_out/y_raw.csv
bench.py reports the entry of its workload from profiles/traffic.json as roofline.traffic."""
import csv
import json
import sys

out = {"_comment": "dram__bytes_read.sum + dram__bytes_write.sum per launch of the dominant kernel, one `ncu --set full "
       "--clock-control none` capture each (tools/ncu_capture.sh); bench.py copies the matching entry into roofline.traffic"}
for arg in sys.argv[2:]:
    wl, path = arg.split("=")
    rows = list(csv.reader(open(path)))
    hdr = rows[0]
    vals = rows[-1]          # rows[1] = units, last = the captured launch
    units = dict(zip(hdr, rows[1]))
    d = dict(zip(hdr, vals))

    def num(key):
        v = float(d[key].replace(",", ""))
        u = units.get(key, "")
        scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "Tbyte": 1e12}.get(u, 1.0)
        return v * scale
    ent = {"kernel": d.get("Kernel Name", "?"), "dram_bytes_read": num("dram__bytes_read.sum"),
           "dram_bytes_write": num("dram__bytes_write.sum"), "source": path}
    for key, name, sc in (("gpu__time_duration.sum", "duration_ms_under_ncu", None),
                          ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active_pct", 1.0),
                          ("sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_fp64_cycles_active_pct", 1.0),
                          ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved_occupancy_pct", 1.0),
                          ("launch__registers_per_thread", "registers_per_thread", 1.0)):
        if key in d:
            v = float(d[key].replace(",", ""))
            if sc is None:
                v *= {"nsecond": 1e-6, "usecond": 1e-3, "msecond": 1.0, "second": 1e3}.get(units.get(key, "msecond"), 1.0)
            ent[name] = v
    out[wl] = ent
json.dump(out, open(sys.argv[1], "w"), indent=1)
print(json.dumps(out, indent=1))
