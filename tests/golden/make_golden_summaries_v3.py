#!/usr/bin/env python
"""Extract the Inter-Area-Prefix origination vectors for the multi-area OSPFv3 snapshots of tests/golden/ospfv3.json
(run in the build container, where the reference sources are; the GPU box has none).  Source (read only):

  holo-ospf/tests/conformance/ospfv3/topologies/<topo>/<rt>/config.json   (each area's type, summary, default-cost)
  tests/golden/ospfv3.json                                                (the router's own Inter-Area-Prefix LSAs)

Per snapshot with more than one area: {"topo", "rt", "router_id", "areas": [{"area_id", "area_type", "summary",
"default_cost", "ranges", "type3": [[prefix, options, metric]], "type4": [[asbr, metric]]}]}, the LSAs being those
the router itself originated into that area as the reference recorded them (compute_net_summaries,
lsa_orig_inter_area_network, holo-ospf ospfv3/lsdb.rs:341-386); options are the recorded option names, sorted.
Output: tests/golden/ospfv3_summaries.json.

Usage: python tests/golden/make_golden_summaries_v3.py [<reference checkout>]
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
AREA_TYPES = {None: "normal", "ietf-ospf:normal-area": "normal", "ietf-ospf:stub-area": "stub",
              "ietf-ospf:nssa-area": "nssa"}


def main(ref: Path):
    topos = ref / "holo-ospf" / "tests" / "conformance" / "ospfv3" / "topologies"
    snaps = json.loads((HERE / "ospfv3.json").read_text())
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
            own = [l for l in a.get("inter_area_lsas", []) if l["adv"] == s["router_id"] and not l.get("maxage")]
            areas.append({
                "area_id": a["area_id"],
                "area_type": AREA_TYPES[c.get("area-type")],
                "summary": bool(c.get("summary", True)),
                "default_cost": int(c.get("default-cost", 10)),   # holo-ietf-ospf-deviations.yang
                "ranges": bool(c.get("ranges")),
                "type3": sorted([l["prefix"], sorted(l.get("options", [])), l["metric"]] for l in own if l["type"] == 3),
                "type4": sorted([l["router_id"], l["metric"]] for l in own if l["type"] == 4),
            })
        out.append({"topo": s["topo"], "rt": s["rt"], "router_id": s["router_id"], "areas": areas})
    (HERE / "ospfv3_summaries.json").write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")
    print(f"{len(out)} snapshots")


if __name__ == "__main__":
    main(Path(sys.argv[1] if len(sys.argv) > 1 else "/root/reference"))
