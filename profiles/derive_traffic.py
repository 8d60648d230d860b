"""Derive profiles/ncu_traffic_r2.json from an ncu launch list + the op sequence recorded by profiles/ncu_frame.py:

  python profiles/derive_traffic.py gpurun_out/launches_c2.csv gpurun_out/opseq_c2.json [out.json]

For the LAST eager frame of the list: DRAM bytes (dram__bytes_read.sum + dram__bytes_write.sum), time under ncu and launch count
per kernel FAMILY (the names bench.py's `roofline.kernels[]` uses), plus the dominant kernel's bytes per launch
(`k_conv2d_tc_bytes_per_launch`, read by bench.py -> `roofline.traffic`).  Numbers taken under ncu are cold-cache and serialised:
they give DRAM bytes and SHARES, never bench values."""
import csv
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SCALE = {"msecond": 1e6, "usecond": 1e3, "nsecond": 1.0, "ns": 1.0, "us": 1e3, "ms": 1e6,
         "Mbyte": 1e6, "Kbyte": 1e3, "Gbyte": 1e9, "byte": 1.0}
OURS = re.compile(r"(k_[a-z0-9_]+|DeviceRadixSort|DeviceScan|cub::)")
# ops that launch a library sort (a variable number of kernels): consume launches while the kernel name belongs to the op
VARIABLE = {"lss_pool_sorted": re.compile(r"(k_lss_|DeviceRadixSort|cub::)"), "box_decode_nms": re.compile(r"(k_decode|k_gather_top|k_iou_mask|k_nms_finish|k_emit|DeviceRadixSort|cub::)")}


def load(path):
    rows = list(csv.reader(l for l in open(path, errors="replace") if l.startswith('"')))
    hdr, data = rows[0], {}
    for r in rows[1:]:
        d = dict(zip(hdr, r))
        try:
            v = float(d["Metric Value"].replace(",", "")) * SCALE.get(d["Metric Unit"], 1.0)
        except ValueError:
            continue
        data.setdefault(int(d["ID"]), {"name": d["Kernel Name"]})[d["Metric Name"]] = v
    return [data[i] for i in sorted(data)]


def byt(l):
    return l.get("dram__bytes_read.sum", 0.0) + l.get("dram__bytes_write.sum", 0.0)


def us(l):
    return l.get("gpu__time_duration.sum", 0.0) / 1e3


def main():
    src, seqf = sys.argv[1], sys.argv[2]
    out_path = sys.argv[3] if len(sys.argv) > 3 else os.path.join(HERE, "ncu_traffic_r2.json")
    launches = load(src)
    seq = json.load(open(seqf))
    # the recorded frame = everything after the LAST first-kernel of the frame's first op
    ours = [l for l in launches if OURS.search(l["name"])]
    # the recorded frame starts at the last launch of the first op's first kernel (e.g. k_cells_insert for lidar workloads)
    first_idx = [i for i, l in enumerate(ours) if "k_cells_insert" in l["name"] or "k_conv2d_dense" in l["name"]]
    need = sum(o["launches"] for o in seq["ops"])
    start = max([i for i in first_idx if len(ours) - i >= need * 0.8] or [max(0, len(ours) - need)])
    frame = ours[start:]
    fam, i = {}, 0
    for o in seq["ops"]:
        d = fam.setdefault(o["family"], {"launches": 0, "us_under_ncu": 0.0, "dram_bytes": 0.0, "kernels": set()})
        if o["family"] in VARIABLE:
            n = 0
            while i + n < len(frame) and VARIABLE[o["family"]].search(frame[i + n]["name"]):
                n += 1
        else:
            n = o["launches"]
        for l in frame[i:i + n]:
            d["launches"] += 1; d["us_under_ncu"] += us(l); d["dram_bytes"] += byt(l)
            m = re.search(r"(k_[a-z0-9_]+|DeviceRadixSort\w*|DeviceScan\w*)", l["name"])
            d["kernels"].add(m.group(1) if m else l["name"][:40])
        i += n
    tot_us = sum(d["us_under_ncu"] for d in fam.values()) or 1.0
    tc = [l for l in frame if "k_conv2d_tc" in l["name"] or "k_gconv3x3_ring" in l["name"]]      # the wgmma dense-map convolutions
    out = {
        "source": f"{os.path.basename(src)} + {os.path.basename(seqf)}: ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,"
                  "dram__bytes_write.sum --clock-control none, python profiles/ncu_frame.py, last eager frame; cold-cache, serialised",
        "workload": seq.get("workload"), "precision": seq.get("precision"),
        "frame_launches": len(frame), "frame_us_under_ncu": sum(map(us, frame)),
        "all_kernels_dram_bytes_per_frame": sum(map(byt, frame)),
        "k_conv2d_tc_launches_per_frame": len(tc),
        "k_conv2d_tc_bytes_per_launch": sum(map(byt, tc)) / max(len(tc), 1),
        "k_conv2d_tc_dram_bytes_per_frame": sum(map(byt, tc)),
        "k_conv2d_tc_share_of_frame_under_ncu": sum(map(us, tc)) / (sum(map(us, frame)) or 1.0),
        "per_family_dram_bytes_per_frame": {k: d["dram_bytes"] for k, d in fam.items()},
        "per_family": {k: {"launches": d["launches"], "us_under_ncu": d["us_under_ncu"], "share_under_ncu": d["us_under_ncu"] / tot_us,
                           "dram_mb": d["dram_bytes"] / 1e6, "kernels": sorted(d["kernels"])} for k, d in
                       sorted(fam.items(), key=lambda kv: -kv[1]["us_under_ncu"])},
    }
    with open(out_path, "w") as fh:
        json.dump(out, fh, indent=1)
    print(json.dumps({k: v for k, v in out.items() if k != "per_family"}, indent=1)[:1500])


if __name__ == "__main__":
    main()
