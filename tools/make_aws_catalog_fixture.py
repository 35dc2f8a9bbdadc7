#!/usr/bin/env python3
"""Derive karpenter_b200/data/aws_instance_types.tsv from the reference's KWOK example catalog
(kwok/examples/aws_instance_types.json of the reference, 1724 entries x 8 offerings; its path is the first argument).

The catalog is benchmark INPUT DATA (SURVEY.md section 8(d): configs C2/C3/C5 use its first 500 / 1000 entries); the
reference tree is not present on the GPU box, so the regular structure (4 zones x {spot, on-demand}, one on-demand and
one spot price per type) is stored as one row per type. The script asserts that regularity so nothing is lost.
Run here (authoring container), commit the output.
"""
import json
import sys

SRC = sys.argv[1]
DST = sys.argv[2] if len(sys.argv) > 2 else "karpenter_b200/data/aws_instance_types.tsv"
ZONES = ["us-west-2a", "us-west-2b", "us-west-2c", "us-west-2d"]

rows = []
for e in json.load(open(SRC)):
    od, spot = set(), set()
    seen = []
    for o in e["offerings"]:
        assert o["Available"] is True and len(o["Requirements"]) == 2
        req = {r["key"]: r for r in o["Requirements"]}
        assert all(r["operator"] == "In" and len(r["values"]) == 1 for r in req.values())
        ct = req["karpenter.sh/capacity-type"]["values"][0]
        zone = req["topology.kubernetes.io/zone"]["values"][0]
        seen.append((ct, zone))
        (od if ct == "on-demand" else spot).add(o["Price"])
    assert seen == [(ct, z) for z in ZONES for ct in ("spot", "on-demand")], seen
    assert len(od) == 1 and len(spot) == 1
    assert len(e["operatingSystems"]) == 1
    r = e["resources"]
    assert set(r) == {"cpu", "memory", "pods", "ephemeral-storage"}
    rows.append([e["name"], e["architecture"], e["operatingSystems"][0], r["cpu"], r["memory"], r["pods"],
                 r["ephemeral-storage"], repr(od.pop()), repr(spot.pop())])
with open(DST, "w") as f:
    f.write("# name\tarch\tos\tcpu\tmemory\tpods\tephemeral-storage\ton_demand_price\tspot_price\n")
    for r in rows:
        f.write("\t".join(r) + "\n")
print(f"wrote {len(rows)} rows to {DST}")
