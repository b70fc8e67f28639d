"""Key numbers of a bench.py JSON line (for the tables in BASELINE.md).  usage: summarize_bench.py file.json [...]"""
import json
import sys

for path in sys.argv[1:]:
    d = json.loads([l for l in open(path) if l.startswith("{")][-1])
    if d.get("impl") == "reference":
        print(path, "reference arm:", round(d["value"], 1), d["unit"], "cores", d["cpu_baseline"]["cores"], "| sample:", d["cpu_baseline"]["sample"][:120])
        continue
    print(path)
    print("  N =", d["n_gpus"], "| value", round(d["value"]), "| one lane", round(d["lanes"]["value_one_lane"]), "| e2e", round(d["e2e"]["value"]),
          "| e2e xyzi", round(d["e2e"].get("value_xyzi_queries", 0)), "| ms/step", round(d["ms_per_step"], 4), "| lanes", d["lanes"]["handles"])
    print("  h2d/d2h bytes per step", d["e2e"]["h2d_bytes_per_step"], d["e2e"]["d2h_bytes_per_step"], "| launches", d["gpu_launches"], "| clocks", d.get("clocks"))
    r = d["roofline"]
    print("  roofline:", r["kernel"], "frac", round(r["frac"], 4), "| by kernel:", {k: (round(1000 * v["avg_launch_ms"], 1), round(v["frac"], 3)) for k, v in r["by_kernel"].items()})
    print("  pipeline:", {k: (round(v, 4) if isinstance(v, float) else v) for k, v in d["pipeline"].items() if k != "note"})
    print("  cpu_baseline:", round(d["cpu_baseline"]["value"], 1), "scans/s on", d["cpu_baseline"]["cores"], "core | quality", d.get("quality_final_map", {}).get("PR"), d.get("quality_final_map", {}).get("RR"))
    if "offline_pass" in d:
        o = d["offline_pass"]
        print("  offline pass:", round(o["ms_per_scan"], 4), "ms/scan,", o["gpu_launches"] // max(1, o["processed_scans"]), "launches/scan, bit-identical", o["final_map_bit_identical_to_oracle"],
              "| oracle", round(o["cpu_oracle_scans_per_s"], 1), "scans/s | passes ms", o["pass_ms"])
    if "exchange" in d:
        print("  exchange:", json.dumps(d["exchange"])[:300])
    if isinstance(d.get("configs"), dict) and isinstance(d["configs"].get("3_seqs_00_01_02_07"), dict):
        print("  config 3:", {k: (round(v["scans_per_s"]), v["PR"], v["RR"]) for k, v in d["configs"]["3_seqs_00_01_02_07"].items()})
