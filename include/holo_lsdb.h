/*
 * holo_lsdb.h — flat, plain-C images of the link-state databases the SPF path
 * reads, and of the tables it writes.  These are the argument types of the
 * LSDB-level entry points (hspf_ospfv2_run_area, hspf_isis_compute_spt, ...):
 * what the reference's run_area()/compute_spt() take from `Area.state.lsdb` /
 * `Lsdb` plus the local interface/neighbour state, restated as arrays so they
 * can cross a C ABI.  The CPU oracle (oracle/*.cc, test infrastructure) consumes
 * the same images, so parity tests feed both sides identical bytes.
 *
 * All addresses / router ids are IPv4 values in host byte order (u32), so
 * numeric order == Ipv4Addr Ord.  Arrays that model a BTreeMap/BTreeSet are
 * documented with the order the producer must supply.
 */
#ifndef HOLO_LSDB_H
#define HOLO_LSDB_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HL_LSA_MAX_AGE 3600u   /* holo-ospf/src/packet/lsa.rs:145-147 is_maxage */

/* ------------------------------------------------------------------ OSPFv2 -- */

/* Router-LSA link types (holo-ospf/src/ospfv2/packet/lsa.rs LsaRouterLinkType) */
#define HL_LINK_P2P     1u
#define HL_LINK_TRANSIT 2u
#define HL_LINK_STUB    3u
#define HL_LINK_VLINK   4u

/* Router-LSA flags (LsaRouterFlags): B=0x01 E=0x02 V=0x04 */
#define HL_RTR_FLAG_B 0x01u
#define HL_RTR_FLAG_E 0x02u
#define HL_RTR_FLAG_V 0x04u

typedef struct hl_ospfv2_link {
    uint32_t link_id;
    uint32_t link_data;
    uint16_t metric;
    uint8_t  link_type;
    uint8_t  _pad;
} hl_ospfv2_link;

/* Router-LSAs, in LsaKey order (adv_rtr, lsa_id) (packet/lsa.rs:44-56). */
typedef struct hl_ospfv2_router_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint16_t age;
    uint8_t  flags;
    uint8_t  options;
    uint32_t link_off;     /* into links[] */
    uint32_t n_links;
} hl_ospfv2_router_lsa;

/* Network-LSAs, in LsaKey order (adv_rtr, lsa_id); attached routers ascending
 * (BTreeSet, ospfv2/spf.rs:398-418). */
typedef struct hl_ospfv2_network_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint32_t mask;
    uint16_t age;
    uint16_t _pad;
    uint32_t att_off;      /* into attached[] */
    uint32_t n_att;
} hl_ospfv2_network_lsa;

/* Interface types (holo-ospf/src/interface.rs InterfaceType + loopback). */
#define HL_IF_P2P       0u
#define HL_IF_BROADCAST 1u
#define HL_IF_NBMA      2u
#define HL_IF_P2MP      3u
#define HL_IF_VLINK     4u
#define HL_IF_LOOPBACK  5u

/* The area's interfaces in NAME order (collections.rs:592: `indexes()` walks
 * name_tree), i.e. the order `nth(link_pos)` counts in (ospfv2/spf.rs:195-201). */
typedef struct hl_ospf_iface {
    uint32_t ifindex;      /* reported in next hops */
    uint32_t sort_key;     /* generational-arena Index order == NexthopKey order
                              (route.rs:92-98); unique per interface            */
    uint8_t  if_type;
    uint8_t  _pad[3];
    uint32_t addr_off;     /* into iface_addrs[]: iface.system.addr_list        */
    uint32_t n_addrs;
    uint32_t nbr_off;      /* into nbrs[]: neighbours of this interface         */
    uint32_t n_nbrs;
} hl_ospf_iface;

typedef struct hl_ipv4_net { uint32_t addr; uint32_t mask; } hl_ipv4_net;
typedef struct hl_ospf_nbr { uint32_t router_id; uint32_t src; } hl_ospf_nbr;

/* SR: Router-Information Opaque LSAs in LsaKey order (adv_rtr, lsa_id); the
 * per-router aggregate follows ospfv2/spf.rs:617-654. */
typedef struct hl_srgb { uint32_t first; uint32_t range; uint8_t first_is_index; uint8_t _pad[3]; } hl_srgb;
typedef struct hl_ospfv2_ri_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint16_t age;
    uint8_t  has_sr_algo;
    uint8_t  sr_algo_has_spf;
    uint32_t srgb_off;     /* into srgbs[] */
    uint32_t n_srgb;
} hl_ospfv2_ri_lsa;

/* Prefix-SID flags (holo-ospf/src/packet/tlv.rs PrefixSidFlags) */
#define HL_PSID_NP 0x40u
#define HL_PSID_M  0x20u
#define HL_PSID_E  0x10u
#define HL_PSID_V  0x08u
#define HL_PSID_L  0x04u

/* Extended-Prefix TLVs of area-scope Extended Prefix Opaque LSAs, flattened in
 * LSDB iteration order (LsaKey order, then TLV order inside the LSA); the first
 * entry per (adv_rtr, prefix) wins (ospfv2/spf.rs:656-689). */
typedef struct hl_ospfv2_ext_prefix {
    uint32_t adv_rtr;
    uint32_t prefix;       /* masked */
    uint32_t mask;
    uint16_t age;
    uint8_t  route_type;   /* ExtPrefixRouteType: 0 unspecified, 1 intra, 3 inter ... */
    uint8_t  has_sid;      /* carries a Prefix-SID for algo SPF */
    uint8_t  sid_flags;
    uint8_t  sid_is_label; /* Sid::Label vs Sid::Index */
    uint8_t  _pad[2];
    uint32_t sid_value;
} hl_ospfv2_ext_prefix;

typedef struct hl_ospfv2_area {
    uint32_t router_id;    /* instance.state.router_id: the SPF root             */
    uint32_t area_id;
    uint16_t max_paths;    /* instance.config.max_paths (default 16)             */
    uint8_t  sr_enabled;
    uint8_t  _pad;
    uint32_t n_router_lsas;  const hl_ospfv2_router_lsa *router_lsas;
    uint32_t n_links;        const hl_ospfv2_link *links;
    uint32_t n_network_lsas; const hl_ospfv2_network_lsa *network_lsas;
    uint32_t n_attached;     const uint32_t *attached;
    uint32_t n_ifaces;       const hl_ospf_iface *ifaces;
    uint32_t n_iface_addrs;  const hl_ipv4_net *iface_addrs;
    uint32_t n_nbrs;         const hl_ospf_nbr *nbrs;
    uint32_t n_ri_lsas;      const hl_ospfv2_ri_lsa *ri_lsas;
    uint32_t n_srgbs;        const hl_srgb *srgbs;
    uint32_t n_ext_prefixes; const hl_ospfv2_ext_prefix *ext_prefixes;
} hl_ospfv2_area;

/* ---- outputs ----------------------------------------------------------------- */

/* Nexthop (route.rs:100-115); `iface` indexes hl_ospfv2_area.ifaces.  Sets of
 * next hops are emitted in NexthopKey order (iface sort_key, then addr with
 * None first). */
typedef struct hl_nexthop {
    uint32_t iface;
    uint32_t addr;
    uint32_t nbr_router_id;
    uint32_t sr_label;
    uint8_t  has_addr;
    uint8_t  has_nbr;
    uint8_t  has_label;
    uint8_t  _pad;
} hl_nexthop;

/* SPT vertex (spf.rs:38-46), emitted in VertexId order (Network < Router). */
typedef struct hl_spt_vertex {
    uint32_t id;           /* dr_addr (network) or router_id (router)            */
    uint32_t distance;
    uint16_t hops;
    uint8_t  is_router;
    uint8_t  _pad;
    uint32_t nh_off;       /* into nexthops[]                                    */
    uint32_t n_nh;
} hl_spt_vertex;

/* Area router table entry (RouteRtr, route.rs:57-66), in router-id order. */
typedef struct hl_route_rtr {
    uint32_t router_id;
    uint32_t metric;
    uint8_t  flags;
    uint8_t  options;
    uint8_t  _pad[2];
    uint32_t nh_off;
    uint32_t n_nh;
} hl_route_rtr;

#define HL_ROUTE_CONNECTED 0x01u   /* RouteNetFlags::CONNECTED */

/* Intra-area network route (RouteNet, route.rs:32-46), in prefix order
 * (Ipv4Network Ord: address, then prefix length). */
typedef struct hl_route_net {
    uint32_t prefix;
    uint32_t mask;
    uint32_t metric;
    uint8_t  flags;
    uint8_t  origin_type;  /* LSA type code of the LS origin: 1 router, 2 network */
    uint8_t  has_prefix_sid;
    uint8_t  has_sr_label;
    uint32_t origin_adv_rtr;
    uint32_t origin_lsa_id;
    uint32_t prefix_sid_value;
    uint8_t  prefix_sid_flags;
    uint8_t  prefix_sid_is_label;
    uint8_t  _pad[2];
    uint32_t sr_label;     /* input label */
    uint32_t nh_off;
    uint32_t n_nh;
} hl_route_net;

/* Caller-allocated result of one run_area + update_rib_intra_area.  *_cap are
 * capacities on input; n_* are the produced counts.  If a capacity is too small
 * the call returns HSPF_E_NOMEM with the required counts filled in. */
typedef struct hl_ospfv2_result {
    uint32_t vertices_cap, n_vertices;   hl_spt_vertex *vertices;
    uint32_t routers_cap,  n_routers;    hl_route_rtr  *routers;
    uint32_t routes_cap,   n_routes;     hl_route_net  *routes;
    uint32_t nexthops_cap, n_nexthops;   hl_nexthop    *nexthops;
    uint8_t  transit_capability;         /* area.state.transit_capability        */
    uint8_t  root_found;                 /* 0: SpfRootNotFound (spf.rs:605-610)  */
    uint8_t  _pad[2];
} hl_ospfv2_result;


/* ----------------------------------------------------------- SPF triggers -- */
/* One LSA whose change scheduled the SPF run (SpfTriggerLsa, holo-ospf/src/spf.rs:115-120): the key and
 * type of `new`.  lsa_type: 1 router, 2 network, 3 summary (network), 4 summary (ASBR), 5 AS-external,
 * 10 area-scope opaque, 11 AS-scope opaque; opaque_type (types 10 / 11): 4 Router-Information,
 * 7 Extended-Prefix, 8 Extended-Link; mask: the body's network mask (types 3 and 5). */
typedef struct hl_lsa_trigger {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint32_t mask;
    uint8_t  lsa_type;
    uint8_t  opaque_type;
    uint8_t  _pad[2];
} hl_lsa_trigger;

/* SpfComputation (spf.rs:123-140, ospfv2/spf.rs:98-171) */
#define HL_SPF_FULL     1u   /* a topological (or SR) change: every area's SPT and the whole table            */
#define HL_SPF_PARTIAL  2u   /* only summary / external LSAs changed: the SPTs stand, the listed destinations
                                are re-examined (update_rib_partial, route.rs:196-340)                        */
typedef struct hl_spf_computation {
    uint32_t kind;                 /* HL_SPF_*                                                               */
    uint32_t n_inter_network;      /* prefixes of changed type-3 LSAs (with_netmask(lsa_id, mask), host bits kept) */
    uint32_t n_inter_router;       /* ASBR ids of changed type-4 LSAs                                          */
    uint32_t n_external;           /* prefixes of changed type-5 LSAs                                          */
    uint32_t cap;                  /* capacity of each of the three arrays below                              */
    hl_ipv4_net *inter_network;    /* sorted, unique (BTreeSet)                                               */
    uint32_t    *inter_router;
    hl_ipv4_net *external;
} hl_spf_computation;

/* ------------------------------------------- batched intra-area route cells -- */
/* One (job, prefix) cell of the device route stage (hspf_ospfv2_routes_batch): what
 * update_rib_intra_area (route.rs:343-446) leaves for that prefix in the SPT of that job, with the
 * next hops still as first-hop atoms (include/holo_spf.h).  Prefixes are those of the area's
 * route table (hspf_ospfv2_rtable_prefixes), in route-table order. */
#define HL_CELL_PRESENT    0x01u   /* the prefix is reachable in this job                                  */
#define HL_CELL_CONNECTED  0x02u   /* RouteNetFlags::CONNECTED: the winner's vertex has hops == 0           */
#define HL_CELL_MIXED_SID  0x04u   /* equal-cost advertisers with different Prefix-SIDs were merged: redo
                                      this job's routes from its planes (hspf_ospfv2_area_from_planes)       */
typedef struct hl_route_cell {
    uint64_t nh_mask;       /* union of the merged advertisers' atom sets                                 */
    uint64_t lasthop_mask;  /* atoms contributed (last) by an advertiser one hop from the root (PHP rule)   */
    uint32_t winner;        /* contributor that defines metric / origin / flags / Prefix-SID (table index)  */
    uint16_t metric;
    uint8_t  flags;         /* HL_CELL_*                                                                   */
    uint8_t  _pad;
} hl_route_cell;

/* ------------------------------------------------ OSPFv2 full routing table -- */
/* Inputs and output of update_rib_full (holo-ospf/src/route.rs:146-193): the stages that
 * follow the per-area SPF — inter-area networks / routers from Summary-LSAs
 * (route.rs:449-533, 653-714), transit areas (route.rs:535-650) and AS-external routes
 * (route.rs:717-827). */
#define HL_LSA_INFINITY 0x00FFFFFFu        /* lsdb.rs:46 */
/* OspfRouteType (holo-utils/src/southbound.rs:86-94), in decreasing preference */
#define HL_PATH_INTRA_AREA      0u
#define HL_PATH_INTER_AREA      1u
#define HL_PATH_TYPE1_EXTERNAL  2u
#define HL_PATH_TYPE2_EXTERNAL  3u

/* Type-3 / type-4 Summary-LSA (ospfv2/spf.rs:539-589), LSDB (LsaKey) order per area. */
typedef struct hl_ospfv2_summary_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;       /* network address (type 3) or ASBR router id (type 4) */
    uint32_t mask;         /* type 3                                               */
    uint32_t metric;
    uint8_t  lsa_type;     /* 3 or 4                                               */
    uint8_t  maxage;
    uint8_t  _pad[2];
} hl_ospfv2_summary_lsa;

/* AS-external-LSA (ospfv2/spf.rs:591-615), instance LSDB order. */
typedef struct hl_ospfv2_external_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint32_t mask;
    uint32_t metric;
    uint32_t fwd_addr;
    uint32_t tag;
    uint8_t  e_bit;        /* type-2 external metric                               */
    uint8_t  maxage;
    uint8_t  _pad[2];
} hl_ospfv2_external_lsa;

/* One attached area, in the order the instance iterates its areas. */
typedef struct hl_ospfv2_rib_area {
    uint32_t area_id;
    uint32_t n_summaries;
    const hl_ospfv2_result      *spf;        /* hspf_ospfv2_run_area output for this area       */
    const hl_ospf_iface         *ifaces;     /* the area's interfaces (next hops index them)     */
    const hl_ospfv2_summary_lsa *summaries;
    uint32_t n_ifaces;
    uint8_t  active;       /* Area::is_active (area.rs:150-156): an interface is not Down         */
    uint8_t  _pad[3];
} hl_ospfv2_rib_area;

/* Route of the merged table, in prefix order.  Next hops are hl_nexthop with `iface` = the
 * interface's sort_key (unique per instance, hl_ospf_iface), in NexthopKey order. */
typedef struct hl_rib_route {
    uint32_t prefix;
    uint32_t mask;
    uint32_t metric;
    uint32_t type2_metric;
    uint32_t tag;
    uint32_t area_id;
    uint8_t  path_type;    /* HL_PATH_*                                            */
    uint8_t  flags;        /* HL_ROUTE_CONNECTED | HL_ROUTE_INSTALLED              */
    uint8_t  has_area;
    uint8_t  has_type2;
    uint32_t nh_off;
    uint32_t n_nh;
    uint32_t sr_label;     /* input label of an intra-area route (from hl_route_net)  */
    uint8_t  has_sr_label;
    uint8_t  _pad[3];
} hl_rib_route;

#define HL_ROUTE_INSTALLED 0x02u   /* RouteNetFlags::INSTALLED (route.rs:50-55) */
#define HL_ROUTE_SUMMARY   0x04u   /* holo-isis RouteFlags::SUMMARY (route.rs:40-46): active L1->L2 summary,
                                      installed as a blackhole route without next hops */

/* One message to the RIB manager produced by update_global_rib (route.rs:833-893). */
#define HL_RIB_INSTALL        1u   /* ibus route_install of new_rib.routes[route]                   */
#define HL_RIB_UNINSTALL      2u   /* new_rib.routes[route] was installed and no longer can be       */
#define HL_RIB_UNINSTALL_OLD  3u   /* old_rib.routes[route]: the prefix is gone from the table       */
typedef struct hl_rib_action {
    uint32_t route;
    uint32_t old_sr_label; /* label of the replaced route (route_install's old_sr_label)             */
    uint8_t  kind;
    uint8_t  has_old_sr_label;
    uint8_t  _pad[2];
} hl_rib_action;

typedef struct hl_ospfv2_rib {
    uint32_t routes_cap,   n_routes;     hl_rib_route *routes;
    uint32_t nexthops_cap, n_nexthops;   hl_nexthop   *nexthops;
} hl_ospfv2_rib;


/* Per-area router tables (area.state.routers, RouteRtr, route.rs:57-66) as update_rib_full leaves them:
 * intra-area entries of the SPF plus inter-area entries from type-4 LSAs.  State carried between a full
 * run and the partial runs that follow it.  Entries in (area order of the call, router id) order; next hops
 * name interfaces by sort key, in NexthopKey order. */
typedef struct hl_rib_rtr {
    uint32_t area_id;
    uint32_t router_id;
    uint32_t metric;
    uint8_t  path_type;    /* HL_PATH_INTRA_AREA / HL_PATH_INTER_AREA */
    uint8_t  flags;        /* HL_RTR_FLAG_* */
    uint8_t  _pad[2];
    uint32_t nh_off;
    uint32_t n_nh;
} hl_rib_rtr;
typedef struct hl_ospfv2_rtr_tables {
    uint32_t rtrs_cap,     n_rtrs;       hl_rib_rtr *rtrs;
    uint32_t nexthops_cap, n_nexthops;   hl_nexthop *nexthops;
} hl_ospfv2_rtr_tables;

/* ------------------------------------------------------------------ OSPFv3 -- */

/* Router-LSA link (holo-ospf/src/ospfv3/packet/lsa.rs LsaRouterLink); link_type uses
 * HL_LINK_P2P / HL_LINK_TRANSIT / HL_LINK_VLINK (OSPFv3 Router-LSAs carry no stub links). */
typedef struct hl_ospfv3_link {
    uint32_t iface_id;
    uint32_t nbr_iface_id;
    uint32_t nbr_router_id;
    uint16_t metric;
    uint8_t  link_type;
    uint8_t  _pad;
} hl_ospfv3_link;

#define HL_V3_OPT_R  0x01u   /* Options::R  */
#define HL_V3_OPT_V6 0x02u   /* Options::V6 */

/* Router-LSA fragments in LsaKey order (adv_rtr, lsa_id): all fragments of one
 * advertising router form ONE vertex (RFC 5340 4.8.1, ospfv3/spf.rs:316-342). */
typedef struct hl_ospfv3_router_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint16_t age;
    uint8_t  flags;        /* HL_RTR_FLAG_* */
    uint8_t  options;      /* HL_V3_OPT_*   */
    uint32_t link_off;
    uint32_t n_links;
} hl_ospfv3_router_lsa;

/* Network-LSAs keyed (adv_rtr, lsa_id = DR interface id); attached routers ascending. */
typedef struct hl_ospfv3_network_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint16_t age;
    uint16_t _pad;
    uint32_t att_off;
    uint32_t n_att;
} hl_ospfv3_network_lsa;

/* IP address / prefix of either family.  Order: IPv4 before IPv6 (IpAddr / IpNetwork
 * derived Ord), then address bytes, then prefix length. */
typedef struct hl_ip_addr { uint8_t bytes[16]; uint8_t is_v6; uint8_t _pad[3]; } hl_ip_addr;

#define HL_PFX_OPT_NU 0x01u   /* PrefixOptions::NU: not used in the routing calculation */
typedef struct hl_ospfv3_prefix {
    hl_ip_addr addr;       /* already masked */
    uint8_t  len;
    uint8_t  options;
    uint16_t metric;
} hl_ospfv3_prefix;

/* SPF triggers of OSPFv3 (SpfTriggerLsa, spf.rs:115-120; Ospfv3::spf_computation_type, ospfv3/spf.rs:96-162).
 * function_code: LsaFunctionCode of `new` — legacy or extended (1/33 router, 2/34 network, 3/35 inter-area-prefix,
 * 4/36 inter-area-router, 5/37 AS-external, 8/40 link, 9/41 intra-area-prefix, 11 grace, 12 router-information).
 * prefixes[prefix_off .. +n_prefixes]: intra-area-prefix: the prefixes of the new AND of the old instance;
 * inter-area-prefix / AS-external: the LSA's prefix.  router_id: inter-area-router: the destination router. */
typedef struct hl_ip_prefix { hl_ip_addr addr; uint8_t len; uint8_t _pad[3]; } hl_ip_prefix;
typedef struct hl_lsa_trigger6 {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint32_t router_id;
    uint32_t prefix_off;
    uint32_t n_prefixes;
    uint16_t function_code;
    uint8_t  _pad[2];
} hl_lsa_trigger6;
typedef struct hl_spf_computation6 {
    uint32_t kind;                 /* HL_SPF_FULL / HL_SPF_PARTIAL                              */
    uint32_t n_intra, n_inter_network, n_inter_router, n_external;
    uint32_t cap;                  /* capacity of each array below                               */
    hl_ip_prefix *intra;           /* sorted, unique (BTreeSet<IpNetwork>: family, address, length) */
    hl_ip_prefix *inter_network;
    uint32_t     *inter_router;
    hl_ip_prefix *external;
} hl_spf_computation6;

/* Intra-Area-Prefix-LSAs in LsaKey order (ospfv3/spf.rs:420-477). */
#define HL_V3_REF_ROUTER  1u
#define HL_V3_REF_NETWORK 2u
typedef struct hl_ospfv3_iap_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint16_t age;
    uint8_t  ref_type;     /* HL_V3_REF_*; 0 = something else (ignored) */
    uint8_t  _pad;
    uint32_t ref_lsa_id;
    uint32_t ref_adv_rtr;
    uint32_t prefix_off;   /* into prefixes[] */
    uint32_t n_prefixes;
} hl_ospfv3_iap_lsa;

/* Link-LSAs of the local interfaces' link-scope LSDBs (ospfv3/spf.rs:592-611). */
typedef struct hl_ospfv3_link_lsa {
    uint32_t iface;        /* index into ifaces[]: whose link-scope LSDB holds it */
    uint32_t adv_rtr;
    uint32_t lsa_id;       /* the neighbour's interface id */
    uint16_t age;
    uint16_t _pad;
    hl_ip_addr linklocal;
} hl_ospfv3_link_lsa;

/* Local interfaces of the area; next hops are found by system ifindex ==
 * Router-LSA link iface_id (get_by_ifindex, ospfv3/spf.rs:187-190). */
typedef struct hl_ospfv3_iface {
    uint32_t ifindex;
    uint32_t sort_key;     /* arena index order (NexthopKey order) */
    uint8_t  if_type;      /* HL_IF_* */
    uint8_t  _pad[3];
} hl_ospfv3_iface;

typedef struct hl_ospfv3_area {
    uint32_t router_id;
    uint32_t area_id;
    uint16_t max_paths;
    uint8_t  af_ipv6;      /* instance address family is IPv6 unicast: V6-bit required */
    uint8_t  _pad;
    uint32_t n_router_lsas;  const hl_ospfv3_router_lsa *router_lsas;
    uint32_t n_links;        const hl_ospfv3_link *links;
    uint32_t n_network_lsas; const hl_ospfv3_network_lsa *network_lsas;
    uint32_t n_attached;     const uint32_t *attached;
    uint32_t n_iap_lsas;     const hl_ospfv3_iap_lsa *iap_lsas;
    uint32_t n_prefixes;     const hl_ospfv3_prefix *prefixes;
    uint32_t n_ifaces;       const hl_ospfv3_iface *ifaces;
    uint32_t n_link_lsas;    const hl_ospfv3_link_lsa *link_lsas;
} hl_ospfv3_area;

typedef struct hl_nexthop6 {
    uint32_t iface;        /* index into hl_ospfv3_area.ifaces */
    uint32_t nbr_router_id;
    hl_ip_addr addr;
    uint8_t  has_addr;
    uint8_t  has_nbr;
    uint8_t  _pad[2];
} hl_nexthop6;

typedef struct hl_spt_vertex6 {   /* VertexId::Network{router_id, iface_id} < Router{router_id} */
    uint32_t router_id;
    uint32_t iface_id;     /* networks only */
    uint32_t distance;
    uint16_t hops;
    uint8_t  is_router;
    uint8_t  _pad;
    uint32_t nh_off;
    uint32_t n_nh;
} hl_spt_vertex6;

typedef struct hl_route_net6 {
    hl_ip_addr prefix;
    uint8_t  len;
    uint8_t  flags;        /* HL_ROUTE_CONNECTED */
    uint8_t  origin_type;  /* 1 router, 2 network */
    uint8_t  prefix_options;
    uint32_t metric;
    uint32_t origin_adv_rtr;
    uint32_t origin_lsa_id;
    uint32_t nh_off;
    uint32_t n_nh;
} hl_route_net6;

/* ---- OSPFv3 full routing table (the same generic stages, route.rs:146-193) ---- */
/* Inter-Area-Prefix-LSA (type 3) / Inter-Area-Router-LSA (type 4), ospfv3/spf.rs:479-526,
 * LSDB (LsaKey) order per area. */
typedef struct hl_ospfv3_inter_area_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint32_t metric;
    uint32_t router_id;    /* type 4: the ASBR                                    */
    hl_ip_addr prefix;     /* type 3                                               */
    uint8_t  len;
    uint8_t  prefix_options;   /* HL_PFX_OPT_NU: skipped (ospfv3/spf.rs:494)      */
    uint8_t  lsa_type;     /* 3 or 4                                               */
    uint8_t  maxage;
} hl_ospfv3_inter_area_lsa;

/* AS-External-LSA (ospfv3/spf.rs:528-560), instance LSDB order. */
typedef struct hl_ospfv3_external_lsa {
    uint32_t adv_rtr;
    uint32_t lsa_id;
    uint32_t metric;
    uint32_t tag;
    hl_ip_addr prefix;
    uint8_t  len;
    uint8_t  prefix_options;
    uint8_t  e_bit;
    uint8_t  maxage;
} hl_ospfv3_external_lsa;

struct hl_ospfv3_result;
typedef struct hl_ospfv3_rib_area {
    uint32_t area_id;
    uint32_t n_summaries;
    const struct hl_ospfv3_result      *spf;      /* hspf_ospfv3_run_area output     */
    const hl_ospfv3_iface              *ifaces;
    const hl_ospfv3_inter_area_lsa     *summaries;
    uint32_t n_ifaces;
    uint8_t  active;
    uint8_t  _pad[3];
} hl_ospfv3_rib_area;

/* Route of the merged table, in prefix order; next hops are hl_nexthop6 with `iface` = the
 * interface's sort_key. */
typedef struct hl_rib_route6 {
    hl_ip_addr prefix;
    uint8_t  len;
    uint8_t  path_type;    /* HL_PATH_*                                            */
    uint8_t  flags;        /* HL_ROUTE_CONNECTED                                   */
    uint8_t  prefix_options;
    uint8_t  has_area;
    uint8_t  has_type2;
    uint8_t  _pad[2];
    uint32_t metric;
    uint32_t type2_metric;
    uint32_t tag;
    uint32_t area_id;
    uint32_t nh_off;
    uint32_t n_nh;
} hl_rib_route6;

typedef struct hl_ospfv3_result {
    uint32_t vertices_cap, n_vertices;   hl_spt_vertex6 *vertices;
    uint32_t routers_cap,  n_routers;    hl_route_rtr   *routers;
    uint32_t routes_cap,   n_routes;     hl_route_net6  *routes;
    uint32_t nexthops_cap, n_nexthops;   hl_nexthop6    *nexthops;
    uint8_t  transit_capability;
    uint8_t  root_found;
    uint8_t  _pad[2];
} hl_ospfv3_result;

typedef struct hl_ospfv3_rib {
    uint32_t routes_cap,   n_routes;     hl_rib_route6 *routes;
    uint32_t nexthops_cap, n_nexthops;   hl_nexthop6   *nexthops;
} hl_ospfv3_rib;

/* ------------------------------------------------------------------- IS-IS -- */

/* LanId / VertexId key: (SystemId as 48-bit big-endian value << 8) | pseudonode.
 * Numeric order == derived Ord of LanId (holo-isis/src/packet/mod.rs:57-67). */
typedef uint64_t hl_lan_id;

#define HL_ISIS_REACH_LEGACY 0u  /* TLV 2  IS reachability, u8 default metric (packet/tlv.rs:263-275)  */
#define HL_ISIS_REACH_EXT    1u  /* TLV 22 extended IS reachability, u32 metric (tlv.rs:277-287)        */
#define HL_ISIS_REACH_MT     2u  /* TLV 222 MT IS reachability, carries mt_id                            */

typedef struct hl_isis_reach {
    hl_lan_id neighbor;
    uint32_t  metric;
    uint16_t  mt_id;
    uint8_t   kind;
    uint8_t   _pad;
} hl_isis_reach;

/* LSP flags needed by the SPF gates (holo-isis/src/spf.rs:556-602) */
#define HL_LSPF_OL             0x01u  /* LspFlags::OL                                            */
#define HL_LSPF_HAS_PROTOCOLS  0x02u  /* Protocols-Supported TLV present                         */
#define HL_LSPF_NLPID_IPV4     0x04u
#define HL_LSPF_NLPID_IPV6     0x08u
#define HL_LSPF_MT_IPV6_OL     0x10u  /* MT entry for topology 2 has MtFlags::OL (pdu.rs:1431-1445) */
#define HL_LSPF_ATT            0x20u  /* LspFlags::ATT (pdu.rs:1414-1428)                        */
#define HL_LSPF_MT_IPV6_ATT    0x40u  /* MT entry for topology 2 has MtFlags::ATT                */

/* LSP fragments in LspId order (lan_id, fragment) (collections.rs:67-74).  Reach
 * entries of a fragment keep TLV order within each kind. */
typedef struct hl_isis_lsp {
    hl_lan_id lan_id;
    uint32_t  seqno;
    uint16_t  rem_lifetime;
    uint8_t   fragment;
    uint8_t   flags;
    uint32_t  reach_off;   /* into reaches[] */
    uint32_t  n_reach;
    uint32_t  ipreach_off; /* into ipreaches[] (route stage only) */
    uint32_t  n_ipreach;
    uint32_t  srgb_off;    /* into srgbs[]: label blocks of the SR-Capabilities sub-TLV (sr.rs:166-256) */
    uint16_t  n_srgb;
    uint8_t   sr_flags;    /* HL_LSP_SR_* */
    uint8_t   flood_algo;  /* first Flooding-Algorithm sub-TLV of the Router Capability TLVs
                              (packet/pdu.rs:1799-1805): 0 = absent, else the algorithm number */
} hl_isis_lsp;

#define HL_ISIS_FLOOD_ZERO_PRUNER    1u   /* FloodingAlgo (packet/iana.rs:249-253) */
#define HL_ISIS_FLOOD_MODIFIED_MANET 2u

/* hl_isis_lsp.sr_flags: first SR-Capabilities / SR-Algorithm sub-TLV of the LSP's Router
 * Capability TLVs (packet/pdu.rs:1785-1797) */
#define HL_LSP_SR_HAS_CAP   0x01u
#define HL_LSP_SR_ALGO_SPF  0x02u  /* an SR-Algorithm sub-TLV is present and lists SPF          */
#define HL_LSP_SR_CAP_V     0x40u  /* SrCapabilitiesFlags::V (MPLS IPv6)                        */
#define HL_LSP_SR_CAP_I     0x80u  /* SrCapabilitiesFlags::I (MPLS IPv4)                        */

/* IP reachability entry of an LSP fragment, TLV order kept within each kind
 * (vertex_networks, holo-isis/src/spf.rs:1141-1281). */
#define HL_ISIS_IP_V4_INTERNAL 0u   /* TLV 128 */
#define HL_ISIS_IP_V4_EXTERNAL 1u   /* TLV 130 */
#define HL_ISIS_IP_V4_EXT      2u   /* TLV 135 extended IPv4 reachability */
#define HL_ISIS_IP_V6          3u   /* TLV 236 */
#define HL_ISIS_IP_MT_V6       4u   /* TLV 237 (mt_id) */
typedef struct hl_isis_ipreach {
    hl_ip_addr prefix;
    uint32_t metric;
    uint16_t mt_id;
    uint8_t  len;
    uint8_t  kind;
    uint8_t  external;     /* TLV 135: prefix-attr X flag; TLV 236/237: external bit */
    uint8_t  has_psid;     /* Prefix-SID sub-TLV for algorithm SPF (spf.rs:1241-1269); TLV 135/236/237 */
    uint8_t  psid_flags;   /* PrefixSidFlags: HL_ISIS_PSID_* (packet/subtlvs/prefix.rs:56-63) */
    uint8_t  psid_is_label;/* Sid::Label (V/L flags) instead of Sid::Index */
    uint32_t psid_value;
} hl_isis_ipreach;

#define HL_ISIS_PSID_R 0x80u
#define HL_ISIS_PSID_N 0x40u
#define HL_ISIS_PSID_P 0x20u
#define HL_ISIS_PSID_E 0x10u
#define HL_ISIS_PSID_V 0x08u
#define HL_ISIS_PSID_L 0x04u

#define HL_ISIS_METRIC_STANDARD 0u   /* MetricType::Standard (narrow) */
#define HL_ISIS_METRIC_WIDE     1u
#define HL_ISIS_METRIC_BOTH     2u
#define HL_ISIS_MT_NONE      0xFFu   /* mt_id: None (flooding topology)  */
#define HL_ISIS_MT_STANDARD  0u
#define HL_ISIS_MT_IPV6      2u
#define HL_ISIS_MODE_NORMAL   0u     /* MetricMode::Normal   */
#define HL_ISIS_MODE_HOPCOUNT 1u     /* MetricMode::HopCount (flooding/manet.rs:59) */

/* An LSP whose installation scheduled the SPF run (spf_sched.trigger_lsps, holo-isis/src/lsdb.rs:1525-1531). */
typedef struct hl_isis_lsp_trigger {
    hl_lan_id lan_id;
    uint8_t   fragment;
    uint8_t   _pad[7];
} hl_isis_lsp_trigger;
#define HL_ISIS_SPF_FULL       1u   /* SpfType::Full (holo-isis/src/spf.rs:148-154): SPTs, flooding cache, routes */
#define HL_ISIS_SPF_ROUTE_ONLY 2u   /* SpfType::RouteOnly: compute_routes over the standing SPTs              */

/* One level's LSDB plus the compute_spt() parameters (spf.rs:525-535). */
typedef struct hl_isis_level {
    uint8_t  metric_type;
    uint8_t  mt_id;
    uint8_t  metric_mode;
    uint8_t  ipv4_enabled;   /* instance.config.is_af_enabled(Ipv4) */
    uint8_t  ipv6_enabled;
    uint8_t  _pad[3];
    uint32_t n_lsps;     const hl_isis_lsp *lsps;
    uint32_t n_reaches;  const hl_isis_reach *reaches;
    uint32_t n_ipreaches; const hl_isis_ipreach *ipreaches;   /* may be 0/NULL for SPT-only calls */
    uint32_t n_srgbs;     const hl_srgb *srgbs;               /* SR label blocks (route stage with SR) */
} hl_isis_level;

/* SPT vertex (Vertex, spf.rs:76-86) in id_tree order (pseudonodes first).
 * parents[] entries index vertices[] of the same result (arena indices in the
 * reference); nexthops[] are the VertexNexthop.system_id values of a
 * `local = false` run, as 48-bit system ids, duplicates and order preserved. */
typedef struct hl_isis_vertex {
    hl_lan_id lan_id;
    uint32_t  distance;
    uint16_t  hops;
    uint16_t  _pad;
    uint32_t  par_off, n_par;
    uint32_t  nh_off,  n_nh;
} hl_isis_vertex;

/* ---- IS-IS local state and the route stage --------------------------------------
 * compute_spt(local = true) resolves first hops through the adjacency arena
 * (resolve_nexthop, spf.rs:948-1002) and compute_routes (spf.rs:838-941) joins the SPT
 * with the IP reachability of every vertex. */
typedef struct hl_isis_adj {
    uint64_t system_id;
    uint8_t  snpa[6];
    uint8_t  up;            /* AdjacencyState::Up */
    uint8_t  level_usage;   /* bit0 L1, bit1 L2 */
    uint8_t  topo_std;      /* adj.topologies contains 0 */
    uint8_t  topo_ipv6;     /* adj.topologies contains 2 */
    uint8_t  has_ipv4;
    uint8_t  has_ipv6;
    uint8_t  area_disjoint; /* adj.area_addrs disjoint from the local ones (instance.rs:575-589) */
    uint8_t  _pad[3];
    uint32_t ipv4;          /* first IPv4 address from the Hello */
    hl_ip_addr ipv6;        /* first IPv6 address */
} hl_isis_adj;

/* Interfaces in NAME order (collections.rs:156-160).  Broadcast interfaces list their LAN
 * adjacencies of the computed level (one per system id); p2p interfaces 0 or 1. */
typedef struct hl_isis_iface {
    uint32_t ifindex;
    uint32_t metric;        /* iface.config.metric.get(level) */
    uint8_t  is_broadcast;
    uint8_t  _pad[3];
    uint32_t adj_off;       /* into adjs[] */
    uint32_t n_adj;
} hl_isis_iface;

typedef struct hl_isis_instance {
    hl_isis_level lvl;      /* lvl.mt_id / lvl.metric_mode are ignored: set per topology */
    uint64_t system_id;     /* instance.config.system_id: the root */
    uint16_t max_paths;
    uint8_t  level;         /* 1 or 2 */
    uint8_t  level_type;    /* 1 = L1 only, 2 = L2 only, 3 = L1/L2 */
    uint8_t  att_ignore;
    uint8_t  mt_ipv6_enabled; /* is_topology_enabled(Ipv6Unicast) */
    uint8_t  sr_enabled;    /* instance.config.sr.enabled: Prefix-SID labels (sr.rs:33-99) */
    uint8_t  _pad;
    uint32_t n_ifaces;  const hl_isis_iface *ifaces;
    uint32_t n_adjs;    const hl_isis_adj *adjs;
} hl_isis_instance;

/* Route nexthop (route.rs:50-61), emitted in BTreeMap<IpAddr, _> order. */
typedef struct hl_isis_nexthop {
    uint64_t system_id;
    uint32_t iface;         /* index into ifaces[] */
    uint32_t sr_label;      /* output label (Nexthop.sr_label) when has_label */
    hl_ip_addr addr;
    uint32_t has_label;     /* 0/1 (a full word: the struct has no hidden bytes) */
} hl_isis_nexthop;

#define HL_ISIS_RT_L2_INTRA 0u   /* IsisRouteType order (holo-utils/src/southbound.rs:99-106) */
#define HL_ISIS_RT_L1_INTRA 1u
#define HL_ISIS_RT_L2_EXT   2u
#define HL_ISIS_RT_L1_EXT   3u

/* Route (route.rs:27-37) in BTreeMap<IpNetwork, Route> order. */
typedef struct hl_isis_route {
    hl_ip_addr prefix;
    uint32_t metric;
    uint8_t  len;
    uint8_t  route_type;
    uint8_t  flags;         /* HL_ROUTE_CONNECTED */
    uint8_t  has_sr_label;
    uint32_t nh_off;
    uint32_t n_nh;
    uint32_t sr_label;      /* input label (Route.sr_label) when has_sr_label */
} hl_isis_route;

/* One configured L1->L2 summary prefix (instance.config.summaries, SummaryCfg:
 * holo-isis/src/northbound/configuration.rs:225-227), and an ACTIVE summary (SummaryRoute,
 * route.rs:72-75): `metric` = the lowest metric of the contributing L1 routes. */
typedef struct hl_isis_summary {
    hl_ip_addr prefix;
    uint32_t cfg_metric;    /* SummaryCfg.metric when has_cfg_metric */
    uint32_t metric;        /* active summaries only: lowest contributing metric */
    uint8_t  len;
    uint8_t  has_cfg_metric;
    uint8_t  _pad[2];
} hl_isis_summary;

typedef struct hl_isis_rib {
    uint32_t routes_cap,   n_routes;    hl_isis_route *routes;
    uint32_t nexthops_cap, n_nexthops;  hl_isis_nexthop *nexthops;
} hl_isis_rib;

/* Remote Neighbor List entry of the modified-MANET flooding reduction (flooding/manet.rs:30-35):
 * BTreeMap<SystemId, FloodingAlgo>, ascending system id. */
typedef struct hl_isis_rnl_entry {
    uint64_t system_id;
    uint8_t  algo;          /* HL_ISIS_FLOOD_* */
    uint8_t  _pad[7];
} hl_isis_rnl_entry;

typedef struct hl_isis_spt {
    uint32_t vertices_cap, n_vertices;  hl_isis_vertex *vertices;
    uint32_t parents_cap,  n_parents;   uint32_t *parents;
    uint32_t nexthops_cap, n_nexthops;  uint64_t *nexthops;
    uint32_t first_hops_cap,  n_first_hops;   uint32_t *first_hops;   /* Spt.first_hops (insertion order)  */
    uint32_t second_hops_cap, n_second_hops;  uint32_t *second_hops;
} hl_isis_spt;

/* One (job, prefix) cell of the IS-IS device route stage (hspf_isis_routes_batch): what compute_routes
 * (holo-isis/src/spf.rs:838-941) leaves for that prefix in the SPT of that job, next hops still as
 * first-hop atoms of the prefix's topology (hspf_atom_decode for the job's root).  Prefixes are those
 * of the instance's route table (hspf_isis_rtable_prefixes), in NetKey order.  flags: HL_CELL_PRESENT,
 * HL_CELL_CONNECTED (the winner's vertex has hops == 0), HL_CELL_MIXED_SID (SR enabled, the route has
 * a Prefix-SID and its best-metric contributions come from two or more vertices: redo this job through
 * hspf_isis_routes_from_planes). */
typedef struct hl_isis_route_cell {
    uint64_t nh_mask;       /* union of the best-metric contributors' atom sets                         */
    uint32_t winner;        /* contributor that set type, CONNECTED and Prefix-SID (table index)        */
    uint32_t metric;        /* distance + entry metric, u32 as compute_routes adds them                 */
    uint8_t  flags;         /* HL_CELL_*                                                                */
    uint8_t  _pad[7];
} hl_isis_route_cell;

/* ------------------------------------------------------------ route deltas -- */
/* What the route-delta stage (hspf_ospfv2_routes_delta, hspf_isis_routes_delta) reports for one (job, prefix)
 * whose cell differs from the job's base cell, compared word for word (for a fixed root, atom numbering does not
 * depend on the job).  B = base cell, J = job cell: */
#define HL_DELTA_LOST      0x01u   /* B is present, J is not                                                   */
#define HL_DELTA_GAINED    0x02u   /* J is present, B is not                                                   */
#define HL_DELTA_METRIC    0x04u   /* both present, the metric differs                                         */
#define HL_DELTA_NEXTHOPS  0x08u   /* both present, nh_mask differs                                            */
#define HL_DELTA_OTHER     0x10u   /* both present, winner or flags differ (OSPF: or lasthop_mask; routing-
                                      table cell: or path type or aux); a new winner can mean a new origin,
                                      route type or SR label                                                   */
typedef struct hl_route_delta {
    uint32_t job;
    uint32_t prefix;        /* index in the route table                                                   */
    uint32_t metric;        /* J's metric; B's when kind is HL_DELTA_LOST                                  */
    uint8_t  kind;          /* HL_DELTA_* (never 0)                                                        */
    uint8_t  _pad[3];
} hl_route_delta;

typedef struct hl_route_delta_job {
    uint32_t n_changed;     /* prefixes with any HL_DELTA_* bit                                           */
    uint32_t n_lost, n_gained, n_metric, n_nexthops, n_other;   /* prefixes carrying that bit            */
    uint32_t status;        /* the job's status word (IS-IS: both topologies'), HSPF_JS_INVALID for a base
                               row out of range; non-zero: not compared, counts 0, no records             */
    uint32_t _pad;
} hl_route_delta_job;

/* ------------------------------------------------------- batched OSPFv2 route-table cells -- */
/* One (job, prefix) cell of the device routing-table stage (hspf_ospfv2_rib_cells): what update_rib_full
 * (route.rs:146-193) leaves for that prefix when the job's root is attached to one area only — intra-area
 * route, else the best inter-area route (type-3), else the best AS-external route (type-5 through the
 * ASBR's entry) — with the next hops still as first-hop atoms.  Prefixes are those of the table
 * (hspf_ospfv2_ribtable_prefixes), in prefix order.  `mpf` packs the metric (bits 0-25: at most
 * 0xFFFE + 2 * 0xFFFFFE, a type-1 external behind a type-4 entry), the HL_PATH_* type (bits 26-27)
 * and the HL_CELL_* flags (bits 28-31). */
typedef struct hl_ospf_rib_cell {
    uint64_t nh_mask;       /* atoms of the winner, equal-cost candidates OR-ed together                  */
    uint64_t aux;           /* intra-area: last-hop atoms (hl_route_cell.lasthop_mask); type-2 external:
                               the type-2 metric; else 0                                                   */
    uint32_t winner;        /* record index in the table, 0xFFFFFFFF: no route                              */
    uint32_t mpf;           /* metric | path type << 26 | flags << 28                                       */
} hl_ospf_rib_cell;
#define HL_RIB_CELL_METRIC_BITS  26u
#define HL_RIB_CELL_METRIC_MAX   0x03FFFFFFu
#define HL_RIB_CELL_MPF(metric, path, flags) \
    ((uint32_t)(metric) | ((uint32_t)(path) << 26) | ((uint32_t)(flags) << 28))
#define HL_RIB_CELL_METRIC(c)    ((c).mpf & HL_RIB_CELL_METRIC_MAX)
#define HL_RIB_CELL_PATH(c)      (((c).mpf >> 26) & 0x3u)
#define HL_RIB_CELL_FLAGS(c)     ((c).mpf >> 28)

#ifdef __cplusplus
}
#endif
#endif /* HOLO_LSDB_H */
