/*
 * holo_spf_lsdb.h — LSDB-level entry points of libholo_spf.so: the calls that
 * replace whole reference functions rather than just their inner loop.
 *
 *   hspf_ospfv2_run_area   <->  run_area<Ospfv2>() + update_rib_intra_area()
 *                               holo-ospf/src/spf.rs:587-729, route.rs:343-446,
 *                               sr.rs:29-77 (as called from compute_spf,
 *                               spf.rs:540-545)
 *   hspf_ospfv2_update_rib_full <-> the stages of update_rib_full() after the SPFs:
 *                               inter-area networks/routers, transit areas, externals
 *                               (route.rs:146-193, 449-827, 895-971); host only
 *   hspf_ospfv2_flatten    <->  the LSDB walk of vertex_lsa_find/vertex_lsa_links
 *                               (ospfv2/spf.rs:356-461) done once, for callers
 *                               that batch many roots / what-if jobs through
 *                               hspf_run_batch (holo_spf.h)
 *
 * The SPT itself (distance, hops, ECMP first-hop sets of every vertex) is always
 * computed by the CUDA kernels; the host code here only flattens the LSDB and maps
 * first-hop atoms back to interface/address next hops, routes and labels.
 */
#ifndef HOLO_SPF_LSDB_H
#define HOLO_SPF_LSDB_H

#include "holo_lsdb.h"
#include "holo_spf.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Flattened OSPFv2 area: CSR + the tables needed to map results back. */
typedef struct hspf_ospfv2_flat hspf_ospfv2_flat;

/* Flatten `area` (host only, no device work).  The image is borrowed for the
 * lifetime of the returned object. */
int hspf_ospfv2_flatten(const hl_ospfv2_area *area, hspf_ospfv2_flat **out);
void hspf_ospfv2_flat_free(hspf_ospfv2_flat *flat);
/* CSR view (pointers owned by `flat`).  saturate_at = 0xFFFF, reject_above =
 * 0xFFFFFFFE, flags = 0. */
int hspf_ospfv2_flat_csr(const hspf_ospfv2_flat *flat, hspf_csr *out);
/* Vertex table: vertex v is Router (is_router[v]=1) router_id / Network dr_addr
 * ids[v].  Arrays of n_vertices entries owned by `flat`. */
int hspf_ospfv2_flat_vertices(const hspf_ospfv2_flat *flat, const uint32_t **ids, const uint8_t **is_router,
                              uint32_t *n_vertices);
/* Per CSR edge: index of the Router-LSA link it came from (into area->links) or
 * 0xFFFFFFFF for Network->Router edges, and the reference's link_pos
 * (ospfv2/spf.rs:440). */
int hspf_ospfv2_flat_edge_tags(const hspf_ospfv2_flat *flat, const uint32_t **link_index, const uint32_t **link_pos);
/* Vertex index of a router id / DR address; 0xFFFFFFFF if it is not a vertex. */
uint32_t hspf_ospfv2_flat_router_vertex(const hspf_ospfv2_flat *flat, uint32_t router_id);
uint32_t hspf_ospfv2_flat_network_vertex(const hspf_ospfv2_flat *flat, uint32_t dr_addr);

/*
 * Full SPF of one area for the local router (area->router_id): flatten, run the
 * SPT on the device, rebuild Vertex.nexthops, the area router table,
 * transit_capability and the intra-area routes (with SR labels when
 * area->sr_enabled).  Returns HSPF_OK, HSPF_E_NOMEM (capacities too small, counts
 * filled in), HSPF_E_NEEDS_ORACLE / HSPF_E_JOB_STATUS (caller must use its CPU
 * path), or another HSPF_E_*.
 */
int hspf_ospfv2_run_area(hspf_ctx *ctx, const hl_ospfv2_area *area, hl_ospfv2_result *out);

/* The post-SPT half of hspf_ospfv2_run_area (Vertex.nexthops, router table, transit_capability,
 * intra-area routes with SR labels) over planes the caller already has — e.g. one job of a
 * what-if batch run through hspf_ospfv2_flatten + hspf_run_batch with area->router_id as root.
 * Planes are indexed by the vertex order of hspf_ospfv2_flatten; nh_words as given to the engine
 * (1..4).  Host only. */
int hspf_ospfv2_area_from_planes(const hl_ospfv2_area *area, const uint32_t *dist, const uint16_t *hops,
                                 const uint64_t *nh_mask, uint32_t nh_words, hl_ospfv2_result *out);

/*
 * Trigger-keyed recomputation (SURVEY 8f: incremental flattener).
 *
 *   hspf_ospfv2_spf_computation_type   Ospfv2::spf_computation_type (holo-ospf/src/ospfv2/spf.rs:98-171):
 *       which work a set of trigger LSAs asks for.  HSPF_E_NOMEM when a set does not fit `cap` (counts filled in).
 *   hspf_ospfv2_flat_update   brings a flattened area up to date with `new_area`, the LSDB image after the
 *       trigger LSAs were installed, touching only what the triggers can have changed:
 *         HSPF_FLAT_UNCHANGED  no trigger bears on the graph (summary / external / opaque LSAs, a refreshed
 *                              Router- or Network-LSA with the same links): the uploaded graph stands;
 *         HSPF_FLAT_COSTS      Router-LSAs changed in link metrics only (an interface cost change): the
 *                              flat's costs are patched in place and edges[] / costs[] list the forward
 *                              CSR edges to hand to hspf_graph_update_costs — nothing else is re-uploaded;
 *         HSPF_FLAT_REBUILT    links appeared or disappeared, a vertex came or went, or the image is laid out
 *                              differently: the flat was rebuilt from scratch; upload it again.
 *       The cost-only shortcut requires new_area to keep the LSAs and links of the old image at the same
 *       indices (same counts, same order), which is what replacing an LSA's body in place gives.  The image
 *       the flat was built from is read during the call (it must still be alive); the flat refers to new_area
 *       afterwards (which must outlive the flat's use).  Stub-link metrics and SR data do
 *       not touch the graph: rebuild the route table (hspf_ospfv2_rtable_create) after any FULL trigger.
 *       HSPF_E_NOMEM: more changed edges than `cap` (n_changed filled in; the flat is already updated).
 */
#define HSPF_FLAT_UNCHANGED 0u
#define HSPF_FLAT_COSTS     1u
#define HSPF_FLAT_REBUILT   2u
int hspf_ospfv2_spf_computation_type(const hl_lsa_trigger *triggers, uint32_t n_triggers, hl_spf_computation *out);
int hspf_ospfv2_flat_update(hspf_ospfv2_flat *flat, const hl_ospfv2_area *new_area, const hl_lsa_trigger *triggers,
                            uint32_t n_triggers, uint32_t *kind, uint32_t *edges, uint32_t *costs, uint32_t cap,
                            uint32_t *n_changed);

/*
 * Partial runs (HL_SPF_PARTIAL): update_rib_partial, holo-ospf/src/route.rs:196-340, OSPFv2.
 *   hspf_ospfv2_rib_router_tables   the per-area router tables a FULL run leaves behind (the same inputs as
 *                                   hspf_ospfv2_update_rib_full): the state the partial runs start from.
 *   hspf_ospfv2_update_rib_partial  only summary / external LSAs changed: the SPTs stand.  The routes of the
 *       named destinations are taken out of the previous table and recomputed from the LSAs into a side table
 *       (inter-area networks, then inter-area routers in the per-area tables, then — when a type-4 LSA changed —
 *       every external route, else the named ones), transit areas are re-examined on the routes that stayed,
 *       update_global_rib runs over the side table against the routes taken out, and the side table is laid over
 *       the previous one.  Like the reference, the recomputed routes do not see the routes that stayed (an
 *       inter-area route recomputed for a prefix that is also intra-area replaces it).
 *       `areas[i].spf` is not read (no SPF ran); `areas[i].summaries`, `.active`, `.area_id`, and
 *       `transit_capability[i]` (area.state.transit_capability of the last SPF) are.
 *       out_rib / out_rtrs: the new state; actions: route indices of out_rib (INSTALL, UNINSTALL) or of prev_rib
 *       (UNINSTALL_OLD).  HSPF_E_NOMEM with the counts filled in when an output is too small.
 */
int hspf_ospfv2_rib_router_tables(uint32_t router_id, const hl_ospfv2_rib_area *areas, uint32_t n_areas,
                                  hl_ospfv2_rtr_tables *out);
int hspf_ospfv2_update_rib_partial(uint32_t router_id, uint32_t max_paths, const hl_ospfv2_rib_area *areas,
                                   const uint8_t *transit_capability, uint32_t n_areas,
                                   const hl_ospfv2_external_lsa *ext, uint32_t n_ext, const hl_spf_computation *partial,
                                   const hl_ospfv2_rib *prev_rib, const hl_ospfv2_rtr_tables *prev_rtrs,
                                   hl_ospfv2_rib *out_rib, hl_ospfv2_rtr_tables *out_rtrs,
                                   hl_rib_action *actions, uint32_t actions_cap, uint32_t *n_actions);

/*
 * Batched intra-area route stage on the device (update_rib_intra_area, holo-ospf/src/route.rs:343-446,
 * for every job of a batch: what-if roots, all routers of an area).
 *
 *   hspf_ospfv2_rtable_create   per flattened area: the area's prefixes in route-table order and, per
 *                               prefix, its advertisers (transit networks, stub links) in the order
 *                               update_rib_intra_area meets them.  Host only; `flat` and its area image
 *                               must outlive the call only.
 *   hspf_ospfv2_rtable_upload   copies the table to the ctx's device.
 *   hspf_ospfv2_routes_batch    one thread per (job, prefix) over DEVICE planes [n_jobs][V] written by
 *   hspf_ospfv2_routes_batch16  hspf_run_batch_async / hspf_run_batch16_async with nh_words == 1:
 *                               cells[n_jobs][P] (device).  `gather_*` (optional) additionally copies
 *                               nh_mask[job][vertex] of listed vertices: the transit networks next to a
 *                               job's root, which the host needs to turn atoms into interfaces.
 *                               Enqueued on the ctx stream behind the batch; no synchronisation.
 *   hspf_ospfv2_run_area_batch  the whole LSDB-level call for a list of root routers: flatten, upload,
 *                               one SPT batch, the route kernel, cells (and status words) back to host
 *                               memory.  cells: [n_roots][P]; P from hspf_ospfv2_rtable_prefixes of a
 *                               table of the same area (returned through *n_prefixes; HSPF_E_NOMEM if
 *                               cells_cap is too small).  A job with a non-zero status word has no valid
 *                               cells (saturation, more than 64 atoms): the caller's single-root path.
 *   hspf_ospfv2_routes_from_cells   host: one job's cells -> the routes / next hops hspf_ospfv2_run_area
 *                               returns for area->router_id (out->routes, out->nexthops; vertices and
 *                               routers are not produced).  `area` carries the root's interface and
 *                               neighbour state and the same LSDB the table was built from.  gather_v /
 *                               gather_nh: nh_mask of the transit networks attached to the root.
 *                               HSPF_E_UNSUPPORTED: a cell is flagged HL_CELL_MIXED_SID, or two atoms
 *                               resolve to the same next hop with different attributes: the cells cannot
 *                               say which advertiser's label a next hop keeps — take this root through
 *                               hspf_ospfv2_run_area (or hspf_ospfv2_area_from_planes over its planes).
 */
typedef struct hspf_ospfv2_rtable hspf_ospfv2_rtable;
int hspf_ospfv2_rtable_create(const hspf_ospfv2_flat *flat, hspf_ospfv2_rtable **out);
void hspf_ospfv2_rtable_free(hspf_ospfv2_rtable *rt);
uint32_t hspf_ospfv2_rtable_prefixes(const hspf_ospfv2_rtable *rt);
uint32_t hspf_ospfv2_rtable_contributors(const hspf_ospfv2_rtable *rt);
/* prefix[P], plen[P], off[P+1]; per contributor: vertex, metric, is_network (any pointer may be NULL) */
int hspf_ospfv2_rtable_arrays(const hspf_ospfv2_rtable *rt, const uint32_t **prefix, const uint32_t **plen,
                              const uint32_t **off, const void **contribs /* 16-byte records, route_cells.h */);
int hspf_ospfv2_rtable_upload(hspf_ctx *ctx, hspf_ospfv2_rtable *rt);
int hspf_ospfv2_routes_batch(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs,
                             const hspf_result *planes, hl_route_cell *cells,
                             uint32_t n_gather, const uint32_t *gather_job, const uint32_t *gather_v,
                             uint64_t *gather_nh);
int hspf_ospfv2_routes_batch16(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs,
                               const hspf_result16 *planes, hl_route_cell *cells,
                               uint32_t n_gather, const uint32_t *gather_job, const uint32_t *gather_v,
                               uint64_t *gather_nh);
int hspf_ospfv2_run_area_batch(hspf_ctx *ctx, const hl_ospfv2_area *area, const uint32_t *root_router_ids,
                               uint32_t n_roots, hl_route_cell *cells, uint64_t cells_cap, uint32_t *n_prefixes,
                               uint32_t *job_status,
                               uint32_t *gather_off /* [n_roots+1] */, uint32_t *gather_v, uint64_t *gather_nh,
                               uint32_t gather_cap, double *device_ms /* [2]: SPT batch, route kernel; may be NULL */);
int hspf_ospfv2_routes_from_cells(const hl_ospfv2_area *area, const hspf_ospfv2_rtable *rt,
                                  const hl_route_cell *cells, const uint32_t *gather_v, const uint64_t *gather_nh,
                                  uint32_t n_gather, hl_ospfv2_result *out);

/*
 * The stages of update_rib_full that follow the per-area SPFs (holo-ospf/src/route.rs:146-193):
 * merges the intra-area routes of the attached areas (route_update / route_compare,
 * route.rs:895-971), adds inter-area network routes and inter-area router entries from the
 * Summary-LSAs (only the backbone's when more than one area is active), re-examines transit
 * areas, and adds AS-external routes through the best ASBR entry.  Pure host table joins over
 * the results of hspf_ospfv2_run_area; no device work.  A prefix that is intra-area in two
 * areas is merged by route_compare; the transit-network overwrite rule (route.rs:387-397)
 * has been applied inside each area and is applied again per route across areas (an area's
 * route whose LS origin is a transit network stays out when its LSA id is lower than the entry's
 * origin, otherwise replaces the entry): per route, not per stub link, because the areas' tables
 * arrive already merged.  Returns HSPF_OK or HSPF_E_NOMEM (counts filled in).
 */
int hspf_ospfv2_update_rib_full(uint32_t router_id, uint32_t max_paths, const hl_ospfv2_rib_area *areas,
                                uint32_t n_areas, const hl_ospfv2_external_lsa *ext, uint32_t n_ext,
                                hl_ospfv2_rib *out);

/*
 * update_global_rib (holo-ospf/src/route.rs:833-893): compares the freshly computed table with
 * the previous one and lists the installs / uninstalls the RIB manager has to see, in the
 * reference's order (new table in prefix order, then vanished prefixes in prefix order).  A route
 * is reinstalled unless metric(), tag, sr_label and the next-hop set are all unchanged; connected
 * routes and routes without next hops are never installed.  `new_rib->routes[].flags` receive
 * HL_ROUTE_INSTALLED as the reference sets it (the next call's `old_rib`).  `old_rib` may be NULL
 * (first computation).  Inter-area routes carry no SR label here (the stage does not run
 * prefix_sid_update for Summary-LSAs).  Host only.
 */
int hspf_ospfv2_rib_diff(const hl_ospfv2_rib *old_rib, hl_ospfv2_rib *new_rib, hl_rib_action *out, uint32_t cap,
                         uint32_t *n_out);
int hspf_ospfv3_rib_diff(const hl_ospfv3_rib *old_rib, hl_ospfv3_rib *new_rib, hl_rib_action *out, uint32_t cap,
                         uint32_t *n_out);

/* The OSPFv3 twin (Inter-Area-Prefix / Inter-Area-Router / AS-External LSAs,
 * holo-ospf/src/ospfv3/spf.rs:479-560; prefixes with the NU option are skipped). */
int hspf_ospfv3_update_rib_full(uint32_t router_id, uint32_t max_paths, const hl_ospfv3_rib_area *areas,
                                uint32_t n_areas, const hl_ospfv3_external_lsa *ext, uint32_t n_ext,
                                hl_ospfv3_rib *out);

/* ---- OSPFv3 ----------------------------------------------------------------
 *   hspf_ospfv3_run_area  <->  run_area<Ospfv3>() + update_rib_intra_area()
 *                              (holo-ospf/src/spf.rs:587-729 with the SpfVersion hooks of
 *                              holo-ospf/src/ospfv3/spf.rs:164-477, route.rs:343-446)
 */
typedef struct hspf_ospfv3_flat hspf_ospfv3_flat;
int hspf_ospfv3_flatten(const hl_ospfv3_area *area, hspf_ospfv3_flat **out);
void hspf_ospfv3_flat_free(hspf_ospfv3_flat *flat);
int hspf_ospfv3_flat_csr(const hspf_ospfv3_flat *flat, hspf_csr *out);
/* The batched route stage for OSPFv3 areas (see "Batched intra-area route stage" above): the table of an OSPFv3
 * area — prefixes of the Intra-Area-Prefix-LSAs in route-table order, advertisers in the order update_rib_intra_area
 * meets them (LSAs in LsaKey order, ospfv3/spf.rs:420-477) — is the same object; upload it with
 * hspf_ospfv2_rtable_upload and run hspf_ospfv2_routes_batch[16] behind hspf_run_batch[16]_async over the area's
 * graph.  hspf_ospfv3_routes_from_cells decodes one job's cells into the routes hspf_ospfv3_run_area returns for
 * area->router_id (out->routes, out->nexthops).  hspf_ospfv3_rtable_prefixes6: the table's prefixes / lengths. */
int hspf_ospfv3_rtable_create(const hspf_ospfv3_flat *flat, hspf_ospfv2_rtable **out);
int hspf_ospfv3_rtable_prefixes6(const hspf_ospfv2_rtable *rt, const hl_ip_addr **prefixes, const uint32_t **lens);
int hspf_ospfv3_routes_from_cells(const hl_ospfv3_area *area, const hspf_ospfv2_rtable *rt, const hl_route_cell *cells,
                                  const uint32_t *gather_v, const uint64_t *gather_nh, uint32_t n_gather,
                                  hl_ospfv3_result *out);
/* Ospfv3::spf_computation_type (holo-ospf/src/ospfv3/spf.rs:96-162): Router-, Network-, Link- and Router-Information
 * LSAs ask for a full run; otherwise the run is partial over the prefixes of the changed Intra-Area-Prefix (old and
 * new instance), Inter-Area-Prefix and AS-external LSAs and the routers of the changed Inter-Area-Router LSAs.
 * HSPF_E_NOMEM when a set does not fit `cap` (counts filled in). */
int hspf_ospfv3_spf_computation_type(const hl_lsa_trigger6 *triggers, uint32_t n_triggers, const hl_ip_prefix *prefixes,
                                     uint32_t n_prefixes, hl_spf_computation6 *out);
/* As hspf_isis_flat_update: the area is re-walked (linear), the flat then describes new_area, and `kind` says what
 * to upload — nothing, the listed edge costs (hspf_graph_update_costs: an interface cost change), or everything. */
int hspf_ospfv3_flat_update(hspf_ospfv3_flat *flat, const hl_ospfv3_area *new_area, uint32_t *kind, uint32_t *edges,
                            uint32_t *costs, uint32_t cap, uint32_t *n_changed);
int hspf_ospfv3_flat_vertices(const hspf_ospfv3_flat *flat, const uint32_t **router_ids, const uint32_t **iface_ids,
                              const uint8_t **is_router, uint32_t *n_vertices);
uint32_t hspf_ospfv3_flat_router_vertex(const hspf_ospfv3_flat *flat, uint32_t router_id);
int hspf_ospfv3_run_area(hspf_ctx *ctx, const hl_ospfv3_area *area, hl_ospfv3_result *out);

/* The post-SPT half of hspf_ospfv3_run_area over caller-supplied planes (see
 * hspf_ospfv2_area_from_planes).  Host only. */
int hspf_ospfv3_area_from_planes(const hl_ospfv3_area *area, const uint32_t *dist, const uint16_t *hops,
                                 const uint64_t *nh_mask, uint32_t nh_words, hl_ospfv3_result *out);

/* ---- IS-IS -------------------------------------------------------------------
 *   hspf_isis_compute_spt  <->  compute_spt(level, root_system_id, local = false,
 *                               mt_id, metric_mode, ..)  holo-isis/src/spf.rs:525-707,
 *                               the call made per MT topology by compute_spf
 *                               (spf.rs:742-757) and per adjacency by
 *                               flooding::manet::init_cache (flooding/manet.rs:47-69)
 *   hspf_isis_flatten + hspf_run_batch + hspf_isis_spt_from_planes: the same, for
 *                               many roots / what-if perturbations per launch.
 */
typedef struct hspf_isis_flat hspf_isis_flat;

int hspf_isis_flatten(const hl_isis_level *lvl, hspf_isis_flat **out);
void hspf_isis_flat_free(hspf_isis_flat *flat);
/* CSR view: reject_above = 1023 / 0xFE000000 by metric type, flags =
 * HSPF_GF_NOHOP_TARGET_NO_NEXTHOP (| HSPF_GF_HOPCOUNT in hop-count mode). */
int hspf_isis_flat_csr(const hspf_isis_flat *flat, hspf_csr *out);
int hspf_isis_flat_vertices(const hspf_isis_flat *flat, const uint64_t **lan_ids, uint32_t *n_vertices);
uint32_t hspf_isis_flat_vertex(const hspf_isis_flat *flat, uint64_t lan_id);
/* Rebuild the reference's Spt (ordered ECMP parents, next-hop Vecs, first/second
 * hops) for one job from its `dist` and `hops` result planes (host pointers). */
int hspf_isis_spt_from_planes(const hspf_isis_flat *flat, uint32_t root_vertex, const uint32_t *dist,
                              const uint16_t *hops, uint32_t n_ov, const uint32_t *ov_edge,
                              const uint32_t *ov_cost, hl_isis_spt *out);
/* One SPT for `root_system_id` (48-bit system id). */
int hspf_isis_compute_spt(hspf_ctx *ctx, const hl_isis_level *lvl, uint64_t root_system_id, hl_isis_spt *out);

/*
 * Trigger-keyed recomputation for IS-IS.
 *   hspf_isis_spf_type     the decision lsp_install makes per installed LSP (holo-isis/src/lsdb.rs:1450-1465,
 *                          1525-1531): a run is FULL when any trigger LSP differs from its previous instance in
 *                          expiry, LSP flags (the image's OL and ATT bits) or its IS-reachability / extended-IS-
 *                          reachability entries (a new LSP always does); otherwise ROUTE_ONLY — compute_routes over the standing SPTs
 *                          (hspf_isis_routes_from_planes with the planes of the last full run).  As in the
 *                          reference, MT IS-reachability (TLV 222) entries are not part of the comparison.
 *   hspf_isis_flat_update  brings a flattened level up to date with `new_lvl` and says what to upload:
 *                          HSPF_FLAT_UNCHANGED / HSPF_FLAT_COSTS (same vertices, edges and flags: only metrics
 *                          moved; edges[] / costs[] for hspf_graph_update_costs) / HSPF_FLAT_REBUILT.  The level
 *                          is re-walked (linear in the LSDB); what is saved is the graph upload.  The flat refers
 *                          to new_lvl afterwards.  HSPF_E_NOMEM: more changed edges than `cap` (n_changed set).
 */
int hspf_isis_spf_type(const hl_isis_level *old_lvl, const hl_isis_level *new_lvl, const hl_isis_lsp_trigger *triggers,
                       uint32_t n_triggers, uint32_t *spf_type);
int hspf_isis_flat_update(hspf_isis_flat *flat, const hl_isis_level *new_lvl, uint32_t *kind, uint32_t *edges,
                          uint32_t *costs, uint32_t cap, uint32_t *n_changed);

/* Route path of one level (compute_spf, holo-isis/src/spf.rs:742-799): for every enabled
 * topology an SPT with `local = true` next-hop resolution (spf.rs:948-1002), then
 * compute_routes (spf.rs:838-941) into one RIB (prefix order). */
int hspf_isis_compute_routes(hspf_ctx *ctx, const hl_isis_instance *inst, hl_isis_rib *out);

/* The same route stage (local next-hop resolution + compute_routes, holo-isis/src/spf.rs:838-1002)
 * over SPT planes the caller already has — e.g. one job of a what-if batch run through
 * hspf_isis_flatten + hspf_run_batch.  `dist_*` / `hops_*` are indexed by the vertex order of
 * hspf_isis_flatten for that topology (lvl.mt_id = HL_ISIS_MT_STANDARD / HL_ISIS_MT_IPV6,
 * lvl.metric_mode = HL_ISIS_MODE_NORMAL) with the local system as root; the IPv6-topology
 * planes are read only when inst->mt_ipv6_enabled.  Host only. */
int hspf_isis_routes_from_planes(const hl_isis_instance *inst, const uint32_t *dist_std, const uint16_t *hops_std,
                                 const uint32_t *dist_mt6, const uint16_t *hops_mt6, hl_isis_rib *out);

/*
 * Batched IS-IS route stage on the device (compute_routes, holo-isis/src/spf.rs:838-941, for every job of a
 * what-if batch).
 *
 *   hspf_isis_rtable_create   per instance: the prefixes of the enabled topologies in NetKey order and, per
 *                             prefix, its contributors in the order compute_routes meets them (vertex order,
 *                             fragments in LspId order, ATT default, TLV 128, 130, 135, 236/237).  Each prefix
 *                             is fed by one topology: IPv4 by the standard one, IPv6 by the standard one or,
 *                             with inst->mt_ipv6_enabled, by MT-IPv6 only.  Vertex numbering per topology is
 *                             that of hspf_isis_flatten with lvl.mt_id set and HL_ISIS_MODE_NORMAL.  Host only;
 *                             `inst` must outlive the call only.
 *   hspf_isis_rtable_topology vertex count and root vertex (0xFFFFFFFF: the root owns no LSP there, or the
 *                             topology is not enabled) of topology 0 (standard) or 1 (MT-IPv6).
 *   hspf_isis_rtable_upload   copies the table to the ctx's device.
 *   hspf_isis_routes_batch    one thread per (job, prefix) over DEVICE planes [n_jobs][V] of each topology
 *   hspf_isis_routes_batch16  written by hspf_run_batch_async / hspf_run_batch16_async with nh_words == 1:
 *                             cells[n_jobs][P] (device).  `mt6` may be NULL unless the table has an MT-IPv6
 *                             root.  A job whose status word is non-zero in either topology gets empty cells.
 *                             Enqueued on the ctx stream behind the batches; no synchronisation.
 *   hspf_isis_routes_from_cells   host: one job's cells -> exactly the hl_isis_rib hspf_isis_routes_from_planes
 *                             returns for the same planes (routes, next hops, SR labels).  dist_* / hops_*: that
 *                             job's planes (the first-hop replay around the root reads them); ov_*: that job's
 *                             edge overrides per topology (HSPF_COST_DISABLED: the edge relaxes nothing), so
 *                             that a what-if job decodes to the routes of an LSDB carrying those metrics.
 *                             HSPF_E_UNSUPPORTED: a cell is flagged HL_CELL_MIXED_SID, or two atoms resolve to
 *                             the same address with different attributes: take this job through
 *                             hspf_isis_routes_from_planes.
 */
typedef struct hspf_isis_rtable hspf_isis_rtable;
int hspf_isis_rtable_create(const hl_isis_instance *inst, hspf_isis_rtable **out);
void hspf_isis_rtable_free(hspf_isis_rtable *rt);
uint32_t hspf_isis_rtable_prefixes(const hspf_isis_rtable *rt);
uint32_t hspf_isis_rtable_contributors(const hspf_isis_rtable *rt);
int hspf_isis_rtable_topology(const hspf_isis_rtable *rt, uint32_t topology, uint32_t *n_vertices, uint32_t *root);
/* prefix[P], len[P], off[P+1], contribs[K] (16-byte records {vertex, metric, topology, external, Prefix-SID
 * present, SR-relevant}, isis_route_cells.h); any pointer may be NULL */
int hspf_isis_rtable_arrays(const hspf_isis_rtable *rt, const hl_ip_addr **prefix, const uint32_t **len,
                            const uint32_t **off, const void **contribs);
int hspf_isis_rtable_upload(hspf_ctx *ctx, hspf_isis_rtable *rt);
int hspf_isis_routes_batch(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result *std_planes,
                           const hspf_result *mt6_planes, hl_isis_route_cell *cells);
int hspf_isis_routes_batch16(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result16 *std_planes,
                             const hspf_result16 *mt6_planes, hl_isis_route_cell *cells);
int hspf_isis_routes_from_cells(const hl_isis_instance *inst, const hspf_isis_rtable *rt, const hl_isis_route_cell *cells,
                                const uint32_t *dist_std, const uint16_t *hops_std,
                                const uint32_t *dist_mt6, const uint16_t *hops_mt6,
                                uint32_t n_ov_std, const uint32_t *ov_edge_std, const uint32_t *ov_cost_std,
                                uint32_t n_ov_mt6, const uint32_t *ov_edge_mt6, const uint32_t *ov_cost_mt6,
                                hl_isis_rib *out);

/*
 * Route-delta stage on the device: which prefixes each job of a what-if batch loses, gains, or reaches at another
 * metric or over another next-hop set, against a base route table — without storing the n_jobs x P cell matrix.
 * Per (job, prefix) it runs the same walk as hspf_*_routes_batch[16] and compares the cell with the job's base cell
 * word for word (for a fixed root, atom a is always the same first hop, whatever the job's overrides).  Enqueued on
 * the ctx stream behind the SPT batches; no synchronisation.
 *
 *   hspf_ospfv2_routes_delta[16]  OSPFv2 and OSPFv3 tables (as hspf_ospfv2_routes_batch[16]).
 *   hspf_isis_routes_delta[16]    IS-IS tables (as hspf_isis_routes_batch[16]).
 *
 *   base_cells  DEVICE [n_base][P] cells, 8-byte aligned: typically written by hspf_*_routes_batch[16] for the
 *               unperturbed job of each root.  n_base == 0 is HSPF_E_INVAL.
 *   base_of     DEVICE [n_jobs] base row of each job, or NULL: every job uses row 0.
 *   job_out     DEVICE [n_jobs] hl_route_delta_job (required).  status: the job's status word (IS-IS: both
 *               topologies' OR-ed), or HSPF_JS_INVALID when base_of[j] >= n_base.  A job with a non-zero status
 *               is not compared: counts 0, no records.
 *   records     DEVICE hl_route_delta[cap], ordered by (job, prefix), identical from run to run.  Only the first
 *               min(total, cap) are written.  records NULL or cap 0: the summaries only.
 *   n_records   DEVICE uint64_t (required): the total number of changed (job, prefix), whatever cap is.
 *
 * Kinds (include/holo_lsdb.h, HL_DELTA_*), with B the base cell and J the job cell: LOST (B present, J not),
 * GAINED (J present, B not); both present: METRIC, NEXTHOPS (nh_mask), OTHER (winner or flags; OSPF: also
 * lasthop_mask) in any combination; neither present: no change.  What is not promised: an unchanged cell does not
 * guarantee unchanged next-hop addresses.  IS-IS addresses come from a replay of the first hops that depends on
 * the order in which the root's neighbours leave the heap; OSPF addresses also read the atom sets of the transit
 * networks attached to the root.  A caller who needs addresses decodes the reported jobs
 * (hspf_*_routes_from_cells).
 */
int hspf_ospfv2_routes_delta(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs, const hspf_result *planes,
                             const hl_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                             hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_ospfv2_routes_delta16(hspf_ctx *ctx, const hspf_ospfv2_rtable *rt, uint32_t n_jobs, const hspf_result16 *planes,
                               const hl_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                               hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_isis_routes_delta(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result *std_planes,
                           const hspf_result *mt6_planes, const hl_isis_route_cell *base_cells, uint32_t n_base,
                           const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                           uint64_t *n_records);
int hspf_isis_routes_delta16(hspf_ctx *ctx, const hspf_isis_rtable *rt, uint32_t n_jobs, const hspf_result16 *std_planes,
                             const hspf_result16 *mt6_planes, const hl_isis_route_cell *base_cells, uint32_t n_base,
                             const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                             uint64_t *n_records);

/* sizeof() of the ABI structs in declaration order (hspf_csr, hspf_jobs,
 * hspf_result, then every struct of holo_lsdb.h); returns the count.  Lets a
 * foreign binding verify its struct layouts at load time. */
/* The end of holo-isis' update_rib (holo-isis/src/route.rs:232-300): the local tables of the two
 * levels are merged, L1 routes preferred (route.rs:236-242), and update_global_rib lists the
 * installs / uninstalls for the RIB manager (a route is reinstalled unless metric and the
 * next-hop set — labels included — are unchanged; connected routes and routes without next hops
 * are never installed; hl_isis_route.flags receive HL_ROUTE_INSTALLED).  Either level may be
 * NULL; `old_rib` may be NULL.  Summary routes (HL_ROUTE_SUMMARY, no next hops) are installed
 * (route.rs:284-288).  Host only. */
int hspf_isis_rib_merge(const hl_isis_rib *l2, const hl_isis_rib *l1, hl_isis_rib *out);
int hspf_isis_rib_diff(const hl_isis_rib *old_rib, hl_isis_rib *new_rib, hl_rib_action *out, uint32_t cap,
                       uint32_t *n_out);

/* L1/L2 routers: summary routes and the L1 -> L2 propagation that uses the L1 SPT distances
 * (SURVEY.md §8f f1; holo-isis/src/route.rs:189-231, lsdb.rs:1149-1357).  Host only.
 *
 *   hspf_isis_summaries        <->  the L1 half of update_rib (route.rs:193-216): every L1 route
 *       covered by a configured summary (shortest-prefix match, JointPrefixMap::get_spm of the
 *       prefix-trie crate) makes that summary active; its metric is the lowest covered metric.
 *       `cfg` in prefix order; `out` (capacity n_cfg) in prefix order.
 *   hspf_isis_rib_add_summaries <-> the L2 half (route.rs:218-229): the active summaries join the
 *       L2 table as routes without next hops, flag HL_ROUTE_SUMMARY, type L2 intra-area, metric =
 *       the configured one if set, else the lowest covered (SummaryRoute::metric).  A summary
 *       replaces an L2 route of the same prefix (BTreeMap::extend).
 *   hspf_isis_l1_to_l2         <->  lsp_propagate_l1_to_l2: the IP reachability of the other
 *       systems' valid non-pseudonode L1 LSPs, metric + L1 SPT distance to the originator
 *       (saturating; narrow TLVs capped at 63), up/down entries and entries covered by a configured
 *       summary left out, the lowest total metric kept per prefix and TLV kind, Prefix-SIDs with
 *       R and P set and E cleared; then one entry per active summary.  `spt_std` / `spt_v6` are
 *       the L1 SPTs of the standard / IPv6-unicast topology (hspf_isis_compute_spt or
 *       hspf_isis_spt_from_planes; spt_v6 NULL: no MT); a system that is not on the SPT
 *       propagates nothing.  `up_down` (may be NULL): one byte per entry of l1->ipreaches, non-zero = the
 *       entry's up/down bit is set.  Output entries ordered by (kind, prefix). */
int hspf_isis_summaries(const hl_isis_rib *l1, const hl_isis_summary *cfg, uint32_t n_cfg, hl_isis_summary *out,
                        uint32_t *n_out);
int hspf_isis_rib_add_summaries(const hl_isis_rib *l2, const hl_isis_summary *active, uint32_t n_active,
                                hl_isis_rib *out);
int hspf_isis_l1_to_l2(const hl_isis_level *l1, const uint8_t *up_down, uint64_t local_system_id,
                       const hl_isis_spt *spt_std, const hl_isis_spt *spt_v6, uint8_t l1_metric_type, uint8_t l2_metric_type,
                       const hl_isis_summary *cfg, uint32_t n_cfg, const hl_isis_summary *active, uint32_t n_active,
                       hl_isis_ipreach *out, uint32_t cap, uint32_t *n_out);

/* ---- IS-IS flooding reduction over the hop-count SPTs of the neighbour batch ------------
 * (SURVEY.md §8f f4; holo-isis/src/flooding/manet.rs).  manet::init_cache runs one hop-count
 * compute_spt per up adjacency (row a16: one hspf_run_batch with HSPF_GF_HOPCOUNT), then per
 * neighbour:
 *   hspf_isis_remote_neighbors  <->  the Remote Neighbor List loop of init_cache (manet.rs:72-88):
 *                                    first hops of the SPT with the flooding algorithm each
 *                                    advertises (default ZeroPruner)
 *   hspf_isis_reflood_list      <->  reflood_list (manet.rs:99-173) with Spt::is_on_path
 *                                    (spf.rs:257-284) and second_hops
 *   hspf_isis_flood_reduction_hash <-> flood_reduction_hash (manet.rs:189-193): Fletcher-16 of the
 *                                    LSP id with fragment >> 3 (crate `fletcher` 1.0)
 * `spt_hopcount` is the hl_isis_spt of the transmitting neighbour (hspf_isis_spt_from_planes /
 * hspf_isis_compute_spt with HL_ISIS_MODE_HOPCOUNT).  Host only. */
uint16_t hspf_isis_flood_reduction_hash(uint64_t lsp_system_id, uint8_t lsp_pseudonode, uint8_t lsp_fragment);
int hspf_isis_remote_neighbors(const hl_isis_level *lvl, const hl_isis_spt *spt_hopcount,
                               hl_isis_rnl_entry *out, uint32_t cap, uint32_t *n_out);
int hspf_isis_reflood_list(const hl_isis_spt *spt_hopcount, const hl_isis_rnl_entry *rnl, uint32_t n_rnl,
                           uint64_t local_system_id, uint64_t lsp_system_id, uint8_t lsp_pseudonode,
                           uint8_t lsp_fragment, uint64_t *out, uint32_t cap, uint32_t *n_out);

int hspf_abi_sizes(uint32_t *out, uint32_t cap);

#ifdef __cplusplus
}
#endif
#endif /* HOLO_SPF_LSDB_H */
