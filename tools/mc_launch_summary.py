"""Per-kernel durations and DRAM bytes of one marching-cubes call per probe volume, from the ncu launch list of
tools/mc_probe.py (ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum -k regex:mc_ --csv).

    python tools/mc_launch_summary.py mc_launches.csv > mc_launches_summary.txt
"""
import collections
import csv
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

KERNELS_PER_CALL = 8      # bits, mark, scan1, compact, eval, scan2, vertex, face
CALLS_PER_VOLUME = 9      # warm-up + 7 timed + 1 with the phase print (tools/mc_probe.py)
VOLUMES = ["257^3 torus", "257^3 dense", "513^3 torus", "513^3 dense"]


def main(path):
    with open(path) as f:
        rows = csv.DictReader([l for l in f if not l.startswith("==")])
        data = collections.OrderedDict()
        for r in rows:
            key = (int(r["ID"]), re.sub(r"\(.*", "", r["Kernel Name"]).replace("<unnamed>::", ""))
            data.setdefault(key, {})[r["Metric Name"]] = float(r["Metric Value"].replace(",", ""))
    peak = bench.peaks()
    items = list(data.items())
    calls = [items[i:i + KERNELS_PER_CALL] for i in range(0, len(items), KERNELS_PER_CALL)]
    print("ncu launch list of tools/mc_probe.py: one call per volume (cold-ish caches, serialised launches); "
          f"HBM peak {peak['hbm']} GB/s from {peak['source']}")
    for vi, name in enumerate(VOLUMES):
        call = calls[vi * CALLS_PER_VOLUME + 5]
        total = sum(m["gpu__time_duration.sum"] for _, m in call) / 1e3
        print(f"\n{name}: {total:.1f} us of kernel time")
        for (_, k), m in call:
            t = m["gpu__time_duration.sum"] / 1e3
            rd, wr = m["dram__bytes_read.sum"] / 1e6, m["dram__bytes_write.sum"] / 1e6
            gbs = (rd + wr) / t * 1e3 if t else 0.0
            print(f"  {k:28s} {t:9.1f} us   DRAM read {rd:8.1f} MB  write {wr:8.1f} MB   {gbs:7.0f} GB/s "
                  f"= {gbs / peak['hbm']:.2f} of the HBM peak")


if __name__ == "__main__":
    main(sys.argv[1])
