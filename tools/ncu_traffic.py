#!/usr/bin/env python3
"""DRAM bytes per frame of the main kernels from `ncu --set full` reports, as JSON on stdout; saved as profiles/traffic.json
(local, git-ignored) it is read by bench.py for roofline.traffic.
    python tools/ncu_traffic.py <frames per launch> <report.ncu-rep> [<report> ...] > profiles/traffic.json
For every kernel the LARGEST launch of each report is taken (the decode kernels also launch an empty repair pass)."""
import csv
import json
import os
import subprocess
import sys

STAGE = {"bc_encode_kernel": "bc_encode", "snappy_encode_fragments_kernel": "snappy_encode", "hap_place_fragments_kernel": "place",
         "snappy_execute_kernel": "snappy_decode", "snappy_index_kernel": "snappy_index", "bc_decode_kernel": "bc_decode"}


def main():
    frames = int(sys.argv[1])
    per = {}
    for rep in sys.argv[2:]:
        out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
        rows = list(csv.reader(out.splitlines()))
        hdr, units, data = rows[0], rows[1], rows[2:]
        ix = {h: i for i, h in enumerate(hdr)}

        def val(r, m):
            v, u = float(r[ix[m]]), units[ix[m]].lower()
            return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(u, 1)
        for r in data:
            name = r[ix["Kernel Name"]].split("(")[0].split("<")[0].replace("hapb200::", "").replace("void ", "").strip()
            st = STAGE.get(name)
            if not st:
                continue
            b = val(r, "dram__bytes_read.sum") + val(r, "dram__bytes_write.sum")
            key = st if "noindex" not in os.path.basename(rep) or st != "snappy_decode" else "snappy_decode_noindex"
            per[key] = max(per.get(key, 0.0), b / frames)
    print(json.dumps({"source": [os.path.basename(r) for r in sys.argv[2:]], "frames_per_launch": frames,
                      "what": "dram__bytes_read.sum + dram__bytes_write.sum per launch / frames (ncu --set full, largest launch of each kernel)",
                      "per_frame_bytes": per}, indent=1))


if __name__ == "__main__":
    main()
