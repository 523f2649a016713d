#!/usr/bin/env python
"""Extract the Summary-LSA origination vectors for the multi-area OSPFv2 snapshots of tests/golden/ospfv2.json
(run in the build container; /root/reference does not exist on the GPU box).  Source (read only):

  holo-ospf/tests/conformance/ospfv2/topologies/<topo>/<rt>/config.json   (each area's type, summary, default-cost)
  tests/golden/ospfv2.json                                                (the router's own type-3 / type-4 LSAs)

Per snapshot with more than one area: {"topo", "rt", "router_id", "areas": [{"area_id", "area_type", "summary",
"default_cost", "ranges", "type3": [[prefix, mask, metric]], "type4": [[asbr, metric]]}]}, the LSAs being those the
router itself originated into that area as the reference recorded them (compute_net_summaries /
compute_rtr_summaries, holo-ospf/src/area.rs:561-740).  Output: tests/golden/ospfv2_summaries.json.

Usage: python tests/golden/make_golden_summaries.py [/root/reference]
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
AREA_TYPES = {None: "normal", "ietf-ospf:normal-area": "normal", "ietf-ospf:stub-area": "stub",
              "ietf-ospf:nssa-area": "nssa"}


def main(ref: Path):
    topos = ref / "holo-ospf" / "tests" / "conformance" / "ospfv2" / "topologies"
    snaps = json.loads((HERE / "ospfv2.json").read_text())
    out = []
    for s in snaps:
        if len(s["areas"]) < 2:
            continue
        cfg = json.loads((topos / s["topo"] / s["rt"] / "config.json").read_text())
        ospf = cfg["ietf-routing:routing"]["control-plane-protocols"]["control-plane-protocol"][0]["ietf-ospf:ospf"]
        conf = {a["area-id"]: a for a in ospf.get("areas", {}).get("area", [])}
        areas = []
        for a in s["areas"]:
            c = conf.get(a["area_id"], {})
            own = [l for l in a["summary_lsas"] if l["adv"] == s["router_id"] and not l["maxage"]]
            areas.append({
                "area_id": a["area_id"],
                "area_type": AREA_TYPES[c.get("area-type")],
                "summary": bool(c.get("summary", True)),
                "default_cost": int(c.get("default-cost", 10)),   # holo-ietf-ospf-deviations.yang
                "ranges": bool(c.get("ranges")),
                "type3": sorted([l["id"], l["mask"], l["metric"]] for l in own if l["type"] == 3),
                "type4": sorted([l["id"], l["metric"]] for l in own if l["type"] == 4),
            })
        out.append({"topo": s["topo"], "rt": s["rt"], "router_id": s["router_id"], "areas": areas})
    (HERE / "ospfv2_summaries.json").write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")
    print(f"{len(out)} snapshots")


if __name__ == "__main__":
    main(Path(sys.argv[1] if len(sys.argv) > 1 else "/root/reference"))
