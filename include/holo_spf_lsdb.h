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
 * Batched routing-table stage on the device, for roots attached to one area (every internal router of the
 * area): update_rib_full (holo-ospf/src/route.rs:146-193) — intra-area, inter-area and AS-external routes —
 * for every job of a batch.  For job j with root router r over area A, the decoded cells of j equal
 *     hspf_ospfv2_update_rib_full(r, A.max_paths, [{A.area_id, spf_j, A.ifaces, summaries, active = 1}], externals)
 * with spf_j = hspf_ospfv2_area_from_planes(A with router_id = r, j's planes): routes and next hops.
 *
 *   hspf_ospfv2_ribtable_create  per flattened area: the prefixes of its intra-area routes, type-3 and type-5
 *                                LSAs (type-3 / type-5 prefixes keep their host bits, as update_rib_full does) in
 *                                prefix order, and per prefix three record ranges: its intra-area advertisers
 *                                (the records of hspf_ospfv2_rtable_create), its type-3 LSAs, its type-5 LSAs, in
 *                                LSDB order.  summaries: the area's type-3 / type-4 LSAs (LsaKey order); externals:
 *                                the instance's AS-external LSAs.  LSAs that no job can use (maxage, metric at
 *                                infinity, a type-3 / type-4 LSA from a router that is not an ABR of the area) are
 *                                left out here.  HSPF_E_UNSUPPORTED when the answer would depend on more than one
 *                                area's SPT: area 0 with a virtual-link endpoint (V flag: the transit-area stage
 *                                could rewrite intra-area routes), or a usable type-4 LSA naming an ABR (its entry
 *                                would replace the ABR's for later type-4 LSAs).  Host only.
 *   hspf_ospfv2_ribtable_arrays  prefix[P], plen[P], off[3 (P + 1)] (intra, type-3, type-5 ranges), the 16-byte
 *                                records (ospf_rib_cells.h); any pointer may be NULL.
 *   hspf_ospfv2_ribtable_upload  copies the table to the ctx's device.
 *   hspf_ospfv2_rib_cells        one thread per (job, prefix) over DEVICE planes as hspf_ospfv2_routes_batch[16],
 *                                for OSPFv2 tables and the OSPFv3 tables of hspf_ospfv3_ribtable_create;
 *   hspf_ospfv2_rib_cells16      roots: device u32[n_jobs], each job's root vertex; cells[n_jobs][P] (device).
 *                                job_status_out (device u32[n_jobs], may be NULL): the planes' status word, plus
 *                                HSPF_JS_INVALID for a root >= V and HSPF_JS_NOT_INTERNAL for a root with the B
 *                                flag (an ABR: its table spans other areas).  A job with a non-zero word gets empty
 *                                cells.  gather_* as hspf_ospfv2_routes_batch.  Enqueued on the ctx stream.
 *   hspf_ospfv2_rib_from_cells   host: one job's cells -> the table above (out->routes in prefix order, next hops
 *                                named by interface sort key in NexthopKey order, HSPF_E_NOMEM with the counts when
 *                                out is too small).  `area` as for hspf_ospfv2_routes_from_cells, with router_id =
 *                                the job's root.  HSPF_E_UNSUPPORTED in the cases of hspf_ospfv2_routes_from_cells:
 *                                take that job through its planes and hspf_ospfv2_update_rib_full.
 *   hspf_ospfv2_rib_delta[16]    what-if batches: each job's cells compared with a base row on the device, without
 *                                storing them (route-delta stage, below).
 */
typedef struct hspf_ospfv2_ribtable hspf_ospfv2_ribtable;
int hspf_ospfv2_ribtable_create(const hspf_ospfv2_flat *flat, uint32_t area_id, const hl_ospfv2_summary_lsa *summaries,
                                uint32_t n_summaries, const hl_ospfv2_external_lsa *externals, uint32_t n_externals,
                                hspf_ospfv2_ribtable **out);
void hspf_ospfv2_ribtable_free(hspf_ospfv2_ribtable *rt);
uint32_t hspf_ospfv2_ribtable_prefixes(const hspf_ospfv2_ribtable *rt);
uint32_t hspf_ospfv2_ribtable_contributors(const hspf_ospfv2_ribtable *rt);
int hspf_ospfv2_ribtable_arrays(const hspf_ospfv2_ribtable *rt, const uint32_t **prefix, const uint32_t **plen,
                                const uint32_t **off, const void **records);
int hspf_ospfv2_ribtable_upload(hspf_ctx *ctx, hspf_ospfv2_ribtable *rt);
int hspf_ospfv2_rib_cells(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result *planes,
                          const uint32_t *roots, hl_ospf_rib_cell *cells, uint32_t *job_status_out,
                          uint32_t n_gather, const uint32_t *gather_job, const uint32_t *gather_v, uint64_t *gather_nh);
int hspf_ospfv2_rib_cells16(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result16 *planes,
                            const uint32_t *roots, hl_ospf_rib_cell *cells, uint32_t *job_status_out,
                            uint32_t n_gather, const uint32_t *gather_job, const uint32_t *gather_v, uint64_t *gather_nh);
int hspf_ospfv2_rib_from_cells(const hl_ospfv2_area *area, const hspf_ospfv2_ribtable *rt, const hl_ospf_rib_cell *cells,
                               const uint32_t *gather_v, const uint64_t *gather_nh, uint32_t n_gather,
                               hl_ospfv2_rib *out);

/*
 * Batched routing-table stage on the device for one area border router (a root with the B flag, which the stage
 * above refuses): update_rib_full over every area the router is attached to, for every job of a what-if batch.
 * One table per router.  Job j holds one row per attached area: rows[j][i] is the row of area i's planes (the
 * SPT of that area's graph rooted at the router).  With attached areas A_0 .. A_{n-1} (flat, area id, type-3/4
 * summaries in LsaKey order, active) and externals X, the decoded cells of job j equal
 *     hspf_ospfv2_update_rib_full(r, max_paths,
 *         [{A_i.area_id, hspf_ospfv2_area_from_planes(A_i, planes_i[rows[j][i]]), A_i.ifaces, summaries_i, active_i}],
 *         X)
 * routes and next hops, with the areas in the caller's order (the instance's area order: it decides the
 * cross-area transit-network rule and the transit-area step) and max_paths the areas' own, which must agree.
 *
 *   hspf_ospfv2_abr_ribtable_create  host.  router_id; per area i < n_areas: flats[i], area_ids[i], summaries[i] /
 *                                n_summaries[i] (n_summaries NULL: none), active[i] (NULL: all active); the
 *                                instance's AS-external LSAs.  Prefixes: the union over the areas, in prefix order;
 *                                per prefix, each area's intra-area advertiser range and type-3 range, and the type-5
 *                                range; per ASBR one entry per area (its vertex with the E flag, its type-4 range,
 *                                which is empty for an area whose summaries step 2 does not read: every area's with
 *                                one active area, else the backbone's); per area its root, its atom base (the atom
 *                                counts of the earlier areas: atom a of area i is bit base_i + a of nh_mask and of an
 *                                intra-area cell's aux) and its V-flag routers.  Filters as hspf_ospfv2_ribtable_create,
 *                                plus the LSAs the router originated itself.  HSPF_E_UNSUPPORTED: more than 8 areas
 *                                (the kernels' bound), more than 64 atoms in all, a usable type-4 LSA naming an ABR in
 *                                an area step 2 reads.  HSPF_E_INVAL: the router is not a router vertex of some flat
 *                                (leave that area out, as update_rib_full callers do when root_found is 0), or the
 *                                areas' max_paths differ.
 *   hspf_ospfv2_abr_ribtable_arrays / _prefixes / _contributors  as for hspf_ospfv2_ribtable (off[(2 n + 1)(P + 1)]:
 *                                per area its intra-area ranges, then per area its type-3 ranges, then the type-5).
 *   hspf_ospfv2_abr_ribtable_areas  per area: root vertex, vertex count, atom base, atom count; returns n_areas.
 *   hspf_ospfv2_abr_ribtable_upload copies the table to the ctx's device.
 *   hspf_ospfv2_abr_rib_cells    one thread per (job, prefix).  planes: host array of n_areas hspf_result (device
 *   hspf_ospfv2_abr_rib_cells16  planes, nh_words == 1) / hspf_result16; n_rows[i] the rows of area i's planes;
 *                                rows: device u32[n_jobs][n_areas]; cells[n_jobs][P] (device) hl_ospf_rib_cell.
 *                                job_status_out (device u32[n_jobs], may be NULL): the OR of the status words of the
 *                                job's rows, plus HSPF_JS_INVALID for a row out of range; a job with a non-zero word
 *                                gets empty cells.  gather_job / gather_area / gather_v (device u32[n_gather]):
 *                                gather_nh[g] = nh_mask of vertex gather_v[g] in the job's row of area gather_area[g]
 *                                (0 when out of range): the transit networks next to the root in each area, which the
 *                                decode reads.  Enqueued on the ctx stream.
 *   hspf_ospfv2_abr_rib_from_cells  host: one job's cells -> the table of the contract.  areas[n_areas]: each area's
 *                                image (router_id = the router), in the table's order; the gathers of the job as
 *                                (area, vertex, nh_mask).  Virtual-link atoms have no next hop, as in
 *                                hspf_ospfv2_area_from_planes; the transit-area step gives such routes theirs.
 *                                HSPF_E_UNSUPPORTED as hspf_ospfv2_rib_from_cells (HL_CELL_MIXED_SID, which also
 *                                marks an intra-area merge across areas or with a transit-area route where a
 *                                Prefix-SID is involved; two atoms with one next hop and different attributes).
 *                                HSPF_E_INVAL for an OSPFv3 table (hspf_ospfv3_abr_rib_from_cells decodes those).
 *   hspf_ospfv2_abr_rib_delta[16]   the route-delta stage over the same walk (arguments as hspf_ospfv2_rib_delta, rows
 *                                as above in place of roots).  The base row is normally the job whose rows are all
 *                                the unperturbed rows.
 */
#define HSPF_ABR_MAX_AREAS 8u
typedef struct hspf_ospfv2_abr_ribtable hspf_ospfv2_abr_ribtable;
int hspf_ospfv2_abr_ribtable_create(uint32_t router_id, uint32_t n_areas, const hspf_ospfv2_flat *const *flats,
                                    const uint32_t *area_ids, const hl_ospfv2_summary_lsa *const *summaries,
                                    const uint32_t *n_summaries, const uint8_t *active,
                                    const hl_ospfv2_external_lsa *externals, uint32_t n_externals,
                                    hspf_ospfv2_abr_ribtable **out);
void hspf_ospfv2_abr_ribtable_free(hspf_ospfv2_abr_ribtable *t);
uint32_t hspf_ospfv2_abr_ribtable_prefixes(const hspf_ospfv2_abr_ribtable *t);
uint32_t hspf_ospfv2_abr_ribtable_contributors(const hspf_ospfv2_abr_ribtable *t);
int hspf_ospfv2_abr_ribtable_arrays(const hspf_ospfv2_abr_ribtable *t, const uint32_t **prefix, const uint32_t **plen,
                                    const uint32_t **off, const void **records);
int hspf_ospfv2_abr_ribtable_areas(const hspf_ospfv2_abr_ribtable *t, uint32_t *root, uint32_t *n_vertices,
                                   uint32_t *atom_base, uint32_t *n_atoms);
int hspf_ospfv2_abr_ribtable_upload(hspf_ctx *ctx, hspf_ospfv2_abr_ribtable *t);
int hspf_ospfv2_abr_rib_cells(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs, const hspf_result *planes,
                              const uint32_t *n_rows, const uint32_t *rows, hl_ospf_rib_cell *cells,
                              uint32_t *job_status_out, uint32_t n_gather, const uint32_t *gather_job,
                              const uint32_t *gather_area, const uint32_t *gather_v, uint64_t *gather_nh);
int hspf_ospfv2_abr_rib_cells16(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs,
                                const hspf_result16 *planes, const uint32_t *n_rows, const uint32_t *rows,
                                hl_ospf_rib_cell *cells, uint32_t *job_status_out, uint32_t n_gather,
                                const uint32_t *gather_job, const uint32_t *gather_area, const uint32_t *gather_v,
                                uint64_t *gather_nh);
int hspf_ospfv2_abr_rib_from_cells(const hspf_ospfv2_abr_ribtable *t, const hl_ospfv2_area *areas, uint32_t n_areas,
                                   const hl_ospf_rib_cell *cells, const uint32_t *gather_area, const uint32_t *gather_v,
                                   const uint64_t *gather_nh, uint32_t n_gather, hl_ospfv2_rib *out);
int hspf_ospfv2_abr_rib_delta(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs, const hspf_result *planes,
                              const uint32_t *n_rows, const uint32_t *rows, const hl_ospf_rib_cell *base_cells,
                              uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                              hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_ospfv2_abr_rib_delta16(hspf_ctx *ctx, const hspf_ospfv2_abr_ribtable *t, uint32_t n_jobs,
                                const hspf_result16 *planes, const uint32_t *n_rows, const uint32_t *rows,
                                const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records);

/*
 * Batched routing-table stage for a backbone router over what-if jobs inside other areas.  R is an internal router
 * of area 0 (no B flag); the "borders" are 1..8 area border routers with area 0 among their areas, each with its
 * ABR table above.  A job changes costs only in the borders' non-backbone areas: R's area-0 SPT is the same in every
 * job (row 0 of R's planes is read) and only the type-3 LSAs the borders originate into area 0 change.  Every area
 * border router of a perturbed area must be given as a border: another one keeps its base type-3 LSAs as static
 * records, and the table cannot tell.  The table
 * holds R's affected prefixes: those with an intra-area record in a non-backbone area of some border.  Every other
 * prefix of R's table is R's base route in every job.  For job j, with border b's ABR cells of j decoded to rib_b
 * (hspf_ospfv2_abr_rib_from_cells), the decoded cells of j equal the affected-prefix routes of
 *     hspf_ospfv2_update_rib_full(R, max_paths, [{0, area_from_planes(area 0, R's row 0), ifaces, S_j, 1}], X)
 * where S_j is area 0's type-3/4 LSAs with each border's type-3 LSAs replaced by hspf_ospfv2_net_summaries(rib_b,
 * target area 0), in LsaKey order.  A border advertises a route of its cell when the cell is present and intra-area,
 * its winner is not one of area 0's intra-area records, no atom is an area-0 atom, and the metric is below
 * LSInfinity.  A border route that ties across areas and whose area-0 next hops max_paths would cut is outside the
 * contract (the cell still counts them).
 *
 *   hspf_ospfv2_backbone_table_create  host.  flat: R's area-0 flat; router_id: R; summaries: area 0's type-3/4 LSAs
 *                                in LsaKey order, as in R's LSDB; externals: the instance's AS-external LSAs; borders:
 *                                the borders' OSPFv2 ABR tables, which must outlive the table.  Per affected prefix:
 *                                R's intra-area records (hspf_ospfv2_ribtable_create's), R's type-3 records with each
 *                                border's LSA replaced by one slot per (border, prefix) at the border's place in
 *                                LsaKey order (also for a border without an LSA for the prefix), and the type-5 range.
 *                                HSPF_E_INVAL: R missing from the flat, R with the B flag or one of the borders, a
 *                                border given twice, a border table without area 0 or for OSPFv3, a border that is
 *                                not a B-flag router vertex of the flat, a usable type-3 LSA of a border for a prefix
 *                                that is not one of its affected prefixes, 0 or more than 8 borders.
 *                                HSPF_E_UNSUPPORTED: area 0 with a V-flag router, a usable type-4 LSA from a border, or
 *                                one naming an ABR (as hspf_ospfv2_ribtable_create).
 *   hspf_ospfv2_backbone_table_prefixes  P, and the prefixes / lengths in prefix order (pointers may be NULL).
 *   hspf_ospfv2_backbone_table_records   the record and slot counts: a slot's winner is n_records + its slot index.
 *   hspf_ospfv2_backbone_table_upload    copies the table to the ctx's device.
 *   hspf_ospfv2_backbone_cells[16]  one thread per (job, prefix).  planes: R's area-0 planes (device, nh_words 1),
 *                                row 0 read; border_cells: host array of n_borders device pointers, border b's cells
 *                                [n_jobs][P_b] in the table's border order (read in place); border_status: host array of
 *                                n_borders device u32[n_jobs] pointers (NULL, or a NULL entry: none).  job_status_out
 *                                (device u32[n_jobs], may be NULL): R's row-0 status word ORed with the borders' job
 *                                words; a job with a non-zero word gets empty cells.  cells[n_jobs][P] (device).
 *                                Nothing is launched for 0 jobs.  Enqueued on the ctx stream.
 *   hspf_ospfv2_backbone_delta[16]  the route-delta stage over the same walk (base cells as hspf_ospfv2_rib_delta).
 *   hspf_ospfv2_backbone_from_cells host: one job's cells -> the table of the contract.  area: R's image of the
 *                                table's area (area 0 here), the one the flat came from; gather_v / gather_nh: nh_mask
 *                                of the transit networks next to R in row 0.  HSPF_E_UNSUPPORTED as hspf_ospfv2_rib_from_cells.
 */
#define HSPF_BACKBONE_MAX_BORDERS 8u
typedef struct hspf_ospfv2_backbone_table hspf_ospfv2_backbone_table;
int hspf_ospfv2_backbone_table_create(const hspf_ospfv2_flat *flat, uint32_t router_id,
                                      const hl_ospfv2_summary_lsa *summaries, uint32_t n_summaries,
                                      const hl_ospfv2_external_lsa *externals, uint32_t n_externals,
                                      const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders,
                                      hspf_ospfv2_backbone_table **out);
void hspf_ospfv2_backbone_table_free(hspf_ospfv2_backbone_table *t);
int hspf_ospfv2_backbone_table_prefixes(const hspf_ospfv2_backbone_table *t, uint32_t *n_prefixes,
                                        const uint32_t **prefix, const uint32_t **plen);
int hspf_ospfv2_backbone_table_records(const hspf_ospfv2_backbone_table *t, uint32_t *n_records, uint32_t *n_slots);
int hspf_ospfv2_backbone_table_upload(hspf_ctx *ctx, hspf_ospfv2_backbone_table *t);
int hspf_ospfv2_backbone_cells(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                               const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                               const uint32_t *const *border_status, uint32_t *job_status_out, hl_ospf_rib_cell *cells);
int hspf_ospfv2_backbone_cells16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, uint32_t *job_status_out, hl_ospf_rib_cell *cells);
int hspf_ospfv2_backbone_delta(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                               const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                               const uint32_t *const *border_status, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                               const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records,
                               uint64_t cap, uint64_t *n_records);
int hspf_ospfv2_backbone_delta16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, const hl_ospf_rib_cell *base_cells,
                                 uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                                 hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_ospfv2_backbone_from_cells(const hspf_ospfv2_backbone_table *t, const hl_ospfv2_area *area,
                                    const hl_ospf_rib_cell *cells, const uint32_t *gather_v, const uint64_t *gather_nh,
                                    uint32_t n_gather, hl_ospfv2_rib *out);

/*
 * The same stage with the borders' type-4 LSAs re-originated per job (OSPFv3: hspf_ospfv3_backbone_asbr_table_create
 * below): a border originates one into
 * area 0 for router A (an ASBR) when A is a router with the E flag in one of its non-backbone areas that it reaches,
 * below LSInfinity, in the job; its metric is that distance (hspf_ospfv2_net_summaries' type-4 rule; an id in two such
 * areas keeps the later area's).  For job j the decoded cells equal the affected-prefix routes of the update_rib_full
 * above, with S_j holding each border's type-3 AND type-4 LSAs from hspf_ospfv2_net_summaries(rib_b, target area 0),
 * in LsaKey order.  R's entry for A is the last usable type-4 LSA, in LsaKey order, whose ABR R reaches (rib_full step
 * 2 replaces the entry per LSA), not the cheapest.  The type-4 rules are restated from the reference's code: no
 * recorded conformance data holds a type-4 or type-5 LSA, so their parity rests on the host restatement alone.
 *
 *   hspf_ospfv2_backbone_asbr_table_create  host.  Arguments as hspf_ospfv2_backbone_table_create; the result may hold
 *                                type-4 slots: per ASBR A some border can originate for, A's type-4 range holds the
 *                                static type-4 records of other ABRs and one slot per (border, non-backbone area where A
 *                                is an E-flag router) at the border's place in LsaKey order (also for a border without
 *                                an LSA for A).  The affected prefixes add every prefix of a usable type-5 LSA of such
 *                                an A.  The refusals of hspf_ospfv2_backbone_table_create apply, except the one of a
 *                                border's type-4 LSA, and: HSPF_E_INVAL a usable type-4 LSA of a border for a router it
 *                                cannot originate for; HSPF_E_UNSUPPORTED a router with the E and the B flag in a
 *                                border's non-backbone area (its entry would replace an ABR's), or slots reading more
 *                                than 8 (border, area) plane sets.
 *   hspf_ospfv2_backbone_table_asbr_slots  the type-4 slot count and the (border, area) plane sets they read (0 and 0
 *                                for a table of hspf_ospfv2_backbone_table_create).  The cells and delta calls above
 *                                refuse a table with type-4 slots (HSPF_E_INVAL), before any launch.
 *   hspf_ospfv2_backbone_asbr_cells[16]  as hspf_ospfv2_backbone_cells[16], plus per border b: border_planes[b] a host
 *                                array of its n_areas plane structs (device, the arrays given hspf_ospfv2_abr_rib_cells,
 *                                same width as `planes`), border_n_rows[b] host u32[n_areas], border_rows[b] device
 *                                u32[n_jobs][n_areas].  Only the plane sets the table's slots name are read.  A job's
 *                                status word also ORs each read row's word; a row out of range gives HSPF_JS_INVALID
 *                                (and empty cells).  For a table without type-4 slots the three arrays may be NULL
 *                                and the output is that of hspf_ospfv2_backbone_cells[16].
 *   hspf_ospfv2_backbone_asbr_delta[16]  the route-delta stage over the same walk.
 * hspf_ospfv2_backbone_from_cells decodes both kinds of table: an external cell's winner is its type-5 record.
 */
int hspf_ospfv2_backbone_asbr_table_create(const hspf_ospfv2_flat *flat, uint32_t router_id,
                                           const hl_ospfv2_summary_lsa *summaries, uint32_t n_summaries,
                                           const hl_ospfv2_external_lsa *externals, uint32_t n_externals,
                                           const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders,
                                           hspf_ospfv2_backbone_table **out);
int hspf_ospfv2_backbone_table_asbr_slots(const hspf_ospfv2_backbone_table *t, uint32_t *n_slots, uint32_t *n_sets);
int hspf_ospfv2_backbone_asbr_cells(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                    const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                    const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                    const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                    uint32_t *job_status_out, hl_ospf_rib_cell *cells);
int hspf_ospfv2_backbone_asbr_cells16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                      const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                      const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                      const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                      uint32_t *job_status_out, hl_ospf_rib_cell *cells);
int hspf_ospfv2_backbone_asbr_delta(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                    const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                    const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                    const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                    const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                    hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                    uint64_t *n_records);
int hspf_ospfv2_backbone_asbr_delta16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                      const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                      const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                      const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                      const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                      hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                      uint64_t *n_records);

/*
 * Non-backbone router over what-if jobs on the backbone (OSPFv3: hspf_ospfv3_nonbackbone_table_create below).  The
 * same stage with source and target area swapped: R is an internal router of a non-backbone area A, and a job
 * changes costs in area 0 only.  R's area-A SPT is its unperturbed one; what changes are the type-3 / type-4 LSAs
 * that A's area border routers attached to area 0 (the "borders") originate into A, because each border's routes
 * move with the job.  The caller must give every area
 * border router of A that is attached to area 0 as a border: another one keeps its base LSAs as static records, and
 * the table cannot tell.  The borders' cells of job j come from hspf_ospfv2_abr_rib_cells[16], with each border's
 * area-0 row of the job and row 0 of its other areas.  For job j, with border b's cells decoded to rib_b, the decoded
 * cells of j equal the affected-prefix routes of
 *     hspf_ospfv2_update_rib_full(R, max_paths, [{A, area_from_planes(A, R's row 0), ifaces, S_j, 1}], X)
 * where S_j is A's type-3/4 LSAs with each border's LSAs replaced by hspf_ospfv2_net_summaries(rib_b, rtrs_b, ...,
 * target A), in LsaKey order.  A border advertises a route of its cell when the cell is present and intra-area or
 * inter-area, its winner is not one of A's intra-area records, no atom is an A atom, and the metric is below
 * LSInfinity.  It originates a type-4 LSA for an ASBR it reaches intra-area, below LSInfinity, in one of its areas
 * other than A (the usual case: an ASBR of area 0, whose distance is read from the border's area-0 row of the job).
 * The affected prefixes are every prefix a border can advertise into A: one with an intra-area record in one of the
 * border's areas other than A, or with a type-3 record in its area 0; with type-4 slots also the prefixes of those
 * ASBRs' type-5 LSAs.  Every other prefix of R's table is R's base route in every job.  In a stub area a border's
 * default route (0.0.0.0/0 at default_cost) stays a static record and no type-4 LSA is originated; a totally stubby
 * area (summary 0) gives a table without slots, possibly with no affected prefix.
 *
 *   hspf_ospfv2_nonbackbone_table_create  host.  flat: R's area-A flat (A is flat's area id); config: A's
 *                                configuration; the other arguments as hspf_ospfv2_backbone_table_create, over A's
 *                                LSDB.  The result is an hspf_ospfv2_backbone_table marked with its target area A;
 *                                the cells and delta calls above (both kinds) and hspf_ospfv2_backbone_table_* take it,
 *                                the table's mark picks the walk, and a table with type-4 slots is the asbr calls', as
 *                                above.  HSPF_E_INVAL: a flat of area 0, a NULL config, R missing from the flat or with
 *                                the B flag, a border given twice or for OSPFv3, a border table without area 0 or A, a
 *                                border that is not a B-flag router vertex of the flat, a usable type-3 LSA of a border
 *                                in A for a prefix it cannot advertise (other than a stub area's default), a usable
 *                                type-4 LSA of a border in A for a router it cannot originate for.
 *                                HSPF_E_UNSUPPORTED: an NSSA, a V-flag router in A (A is a transit area), a usable
 *                                type-4 LSA of another ABR in a border's area-0 summaries (an inter-area router entry
 *                                at the border, whose per-job re-origination is not modelled), a router with the E and
 *                                the B flag in a border's area other than A, slots reading more than 8 (border, area)
 *                                plane sets, 0 or more than 8 borders.
 * hspf_ospfv2_backbone_from_cells decodes the table over R's image of A.
 */
int hspf_ospfv2_nonbackbone_table_create(const hspf_ospfv2_flat *flat, uint32_t router_id,
                                         const struct hl_ospf_area_config *config,
                                         const hl_ospfv2_summary_lsa *summaries, uint32_t n_summaries,
                                         const hl_ospfv2_external_lsa *externals, uint32_t n_externals,
                                         const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders,
                                         hspf_ospfv2_backbone_table **out);

/*
 * Area border router over what-if jobs inside an area it is not attached to.  R is an ABR of area 0 and at least one
 * more active area; a job changes costs only inside another area, whose ABRs attached to area 0 are the "borders"
 * (1..8, each with its ABR table above).  Contract: the jobs perturb no area R is attached to, so each of R's per-area
 * SPTs is row 0 in every job.  Every ABR of the perturbed area attached to area 0 must be given as a border: another
 * one keeps its base LSAs as static records, and the table cannot tell.  update_rib_full at R (more than one active
 * area) reads inter-area routes from area 0's type-3 LSAs only, and ASBR entries of the perturbed area's ASBRs from
 * the borders' type-4 LSAs in area 0; both move with the job, R's intra-area routes do not.  The table holds R's
 * affected prefixes: those some border can advertise into area 0 (an intra-area record in one of its non-backbone
 * areas), and those of a usable type-5 LSA of an ASBR some border can originate a type-4 LSA for.  Every other prefix
 * of R's table is R's base route in every job.  For job j, with border b's ABR cells of j decoded to rib_b, the
 * decoded cells of j equal the affected-prefix routes of
 *     hspf_ospfv2_update_rib_full(R, max_paths, [{A_i.area_id, area_from_planes(A_i, R's row 0 of A_i), ifaces,
 *         S_i, active_i}], X)
 * where S_i is area i's type-3/4 LSAs, area 0's with each border's type-3 and type-4 LSAs replaced by
 * hspf_ospfv2_net_summaries(rib_b, rtrs_b, ..., target area 0), in LsaKey order.  The type-3 rule is the backbone
 * table's, the type-4 rule the asbr table's.
 *
 *   hspf_ospfv2_abr_backbone_table_create  host.  The arguments of hspf_ospfv2_abr_ribtable_create (R's areas in
 *                                instance order; area 0's summaries as in R's LSDB, borders' LSAs included), plus the
 *                                borders' OSPFv2 ABR tables, which must outlive the table.  Per affected prefix: R's
 *                                records as hspf_ospfv2_abr_ribtable_create's, with area 0's type-3 range holding one
 *                                slot per (border, prefix) and each type-4 range of an ASBR some border can originate
 *                                for one slot per (border, non-backbone area where the ASBR is an E-flag router), at
 *                                the borders' LsaKey places.  The refusals of hspf_ospfv2_abr_ribtable_create apply,
 *                                and: HSPF_E_INVAL R not a B-flag router vertex of its area-0 flat, area 0 missing or
 *                                inactive, fewer than two active areas, R one of the borders, a border given twice,
 *                                for OSPFv3, without area 0 or not a B-flag router vertex of R's area-0 flat, a usable
 *                                type-3 / type-4 LSA of a border in area 0 it cannot originate, 0 or more than 8
 *                                borders; HSPF_E_UNSUPPORTED a V-flag router in any of R's areas, a router with the E
 *                                and the B flag in a border's non-backbone area, type-4 slots reading more than 8
 *                                (border, area) plane sets, winners that do not fit.
 *   hspf_ospfv2_abr_backbone_table_prefixes  P, and the prefixes / lengths in prefix order (pointers may be NULL).
 *   hspf_ospfv2_abr_backbone_table_records   the record, slot, type-4 slot and plane-set counts: a slot's winner is
 *                                n_records + its slot index (an OSPFv3 table's, hspf_ospfv3_abr_backbone_table_create:
 *                                n_records + (slot index << 8 | prefix options)).
 *   hspf_ospfv2_abr_backbone_table_upload    copies the table to the ctx's device.
 *   hspf_ospfv2_abr_backbone_cells[16]  one thread per (job, prefix).  planes: host array of R's n_areas plane structs
 *                                (device, as given hspf_ospfv2_abr_rib_cells), row 0 read; border_cells /
 *                                border_status as hspf_ospfv2_backbone_cells; border_planes / border_n_rows /
 *                                border_rows as hspf_ospfv2_backbone_asbr_cells (NULL for a table without type-4
 *                                slots).  job_status_out (device u32[n_jobs], may be NULL): the OR of R's row-0 words,
 *                                the borders' job words and the words of the type-4 rows the job reads, with
 *                                HSPF_JS_INVALID for a row out of range; a job with a non-zero word gets empty cells.
 *                                cells[n_jobs][P] (device).  Nothing is launched for 0 jobs.  Enqueued on the ctx
 *                                stream.
 *   hspf_ospfv2_abr_backbone_delta[16]  the route-delta stage over the same walk (base cells as hspf_ospfv2_rib_delta).
 *   hspf_ospfv2_abr_backbone_from_cells host: one job's cells -> exactly the routes of the affected prefixes of the
 *                                contract.  areas / gathers as hspf_ospfv2_abr_rib_from_cells, of R's row 0.
 *                                HSPF_E_INVAL for an OSPFv3 table (hspf_ospfv3_abr_backbone_from_cells decodes those).
 */
typedef struct hspf_ospfv2_abr_backbone_table hspf_ospfv2_abr_backbone_table;
int hspf_ospfv2_abr_backbone_table_create(uint32_t router_id, uint32_t n_areas, const hspf_ospfv2_flat *const *flats,
                                          const uint32_t *area_ids, const hl_ospfv2_summary_lsa *const *summaries,
                                          const uint32_t *n_summaries, const uint8_t *active,
                                          const hl_ospfv2_external_lsa *externals, uint32_t n_externals,
                                          const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders,
                                          hspf_ospfv2_abr_backbone_table **out);
void hspf_ospfv2_abr_backbone_table_free(hspf_ospfv2_abr_backbone_table *t);
int hspf_ospfv2_abr_backbone_table_prefixes(const hspf_ospfv2_abr_backbone_table *t, uint32_t *n_prefixes,
                                            const uint32_t **prefix, const uint32_t **plen);
int hspf_ospfv2_abr_backbone_table_records(const hspf_ospfv2_abr_backbone_table *t, uint32_t *n_records,
                                           uint32_t *n_slots, uint32_t *n_asbr_slots, uint32_t *n_asbr_sets);
int hspf_ospfv2_abr_backbone_table_upload(hspf_ctx *ctx, hspf_ospfv2_abr_backbone_table *t);
int hspf_ospfv2_abr_backbone_cells(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                   const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                   uint32_t *job_status_out, hl_ospf_rib_cell *cells);
int hspf_ospfv2_abr_backbone_cells16(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                     const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                     const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                     const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                     uint32_t *job_status_out, hl_ospf_rib_cell *cells);
int hspf_ospfv2_abr_backbone_delta(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const hspf_result *const *border_planes,
                                   const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                   const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                   hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                   uint64_t *n_records);
int hspf_ospfv2_abr_backbone_delta16(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                     const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                     const uint32_t *const *border_status, const hspf_result16 *const *border_planes,
                                     const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                     const hl_ospf_rib_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                                     hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap,
                                     uint64_t *n_records);
int hspf_ospfv2_abr_backbone_from_cells(const hspf_ospfv2_abr_backbone_table *t, const hl_ospfv2_area *areas,
                                        uint32_t n_areas, const hl_ospf_rib_cell *cells, const uint32_t *gather_area,
                                        const uint32_t *gather_v, const uint64_t *gather_nh, uint32_t n_gather,
                                        hl_ospfv2_rib *out);

/*
 * The ASBR entries of an area border router C of the table above, per job, for a router of another area of C's
 * (OSPFv2).  When the perturbed area holds an ASBR A, C's area-0 entry for A is inter-area, through the borders'
 * type-4 LSAs in area 0, and C re-originates it into its normal areas other than area 0 (compute_rtr_summaries: E
 * flag, below LSInfinity) at a metric that moves with the job.  The "groups" are the ASBRs whose area-0 type-4 range in
 * C's table holds type-4 slots.
 *
 *   hspf_ospfv2_abr_backbone_table_asbrs  the group count G and the groups' ASBR ids, ascending by group (pointer may
 *                                be NULL).  HSPF_E_INVAL for no table.
 *   hspf_ospfv2_abr_backbone_asbr_entries[16]  one thread per (job, group).  planes, border_planes, border_n_rows and
 *                                border_rows as hspf_ospfv2_abr_backbone_cells[16].  entries (device u32
 *                                [n_jobs][G]): C's area-0 entry metric for the group's ASBR in the job, the metric
 *                                of the type-4 LSA C originates for it into a normal area, or 0xFFFFFFFF when C
 *                                originates none: the type-4 rows of hspf_ospfv2_net_summaries(rib_C, rtrs_C, ...,
 *                                target a normal area other than area 0) over C's routing table of the job.
 *                                job_status_out (device u32[n_jobs], may be NULL): the OR of C's row-0 words and the
 *                                words of the type-4 rows the job reads, HSPF_JS_INVALID for a row out of range; a job
 *                                with a non-zero word gets 0xFFFFFFFF entries.  HSPF_E_INVAL: an OSPFv3 table
 *                                (hspf_ospfv3_abr_backbone_asbr_entries[16] takes those), a table not uploaded,
 *                                entries or job_status_out not 4-byte aligned.  Nothing is launched for 0 jobs.
 *                                Enqueued on the ctx stream.
 */
int hspf_ospfv2_abr_backbone_table_asbrs(const hspf_ospfv2_abr_backbone_table *t, uint32_t *n_groups,
                                         const uint32_t **asbr_ids);
int hspf_ospfv2_abr_backbone_asbr_entries(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                          const hspf_result *planes, const hspf_result *const *border_planes,
                                          const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                          uint32_t *job_status_out, uint32_t *entries);
int hspf_ospfv2_abr_backbone_asbr_entries16(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                            const hspf_result16 *planes, const hspf_result16 *const *border_planes,
                                            const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                            uint32_t *job_status_out, uint32_t *entries);

/*
 * Non-backbone router over what-if jobs inside another non-backbone area (OSPFv2).  R is an internal router of a
 * non-backbone area A2; a job changes costs only inside another non-backbone area A1.  The "borders" are A2's area
 * border routers attached to area 0 (C, 1..8), none attached to A1, each given as its hspf_ospfv2_abr_backbone_table
 * over A1's ABRs attached to area 0 (B).  Every ABR of A2 attached to area 0 must be given as a border: another one
 * keeps its base LSAs as static records, and the table cannot tell.  R's area-A2 SPT is row 0 in every job.  What
 * moves are the type-3 / type-4 LSAs the C's originate into A2: each C's routes move with the B's LSAs in area 0.  For
 * job j, with C's cells of j (hspf_ospfv2_abr_backbone_cells[16]) decoded to rib_C, the decoded cells of j equal the
 * affected-prefix routes of
 *     hspf_ospfv2_update_rib_full(R, max_paths, [{A2, area_from_planes(A2, R's row 0), ifaces, S_j, 1}], X)
 * where S_j is A2's type-3/4 LSAs with each C's LSAs replaced by hspf_ospfv2_net_summaries(rib_C, rtrs_C, ..., target
 * A2), in LsaKey order.  A C's type-3 LSA can move only for a prefix of C's table (C's affected prefixes); any other
 * LSA of C stays a static record.  A C advertises a route of its cell as into a non-backbone area above.  When A1
 * holds an ASBR A, each C's type-4 LSA for A into a normal A2 moves too: in R's type-4 range for A it is a chain slot
 * at C's LsaKey place, which reads C's entries of the job (hspf_ospfv2_abr_backbone_asbr_entries[16]), and the
 * prefixes of A's type-5 LSAs are affected.  The affected prefixes are every prefix of some C's table that C can
 * advertise into A2, plus those.  Every other prefix of R's table is R's base route in every job.  Stub and totally
 * stubby areas are handled as by hspf_ospfv2_nonbackbone_table_create; the chain rule is restated from the reference's
 * code: no recorded conformance data holds a type-4 LSA.
 *
 *   hspf_ospfv2_third_area_table_create  host.  flat: R's area-A2 flat; config: A2's configuration; summaries: A2's
 *                                type-3/4 LSAs in LsaKey order; externals: the AS-external LSAs; borders: the C's
 *                                OSPFv2 abr_backbone tables, which must outlive the table.  The result is an
 *                                hspf_ospfv2_backbone_table marked as a third-area table: hspf_ospfv2_backbone_table_*
 *                                (asbr_slots: the chain slot count and 0 plane sets), _upload and
 *                                hspf_ospfv2_backbone_from_cells take it.  HSPF_E_INVAL: a flat of area 0, a NULL
 *                                config, R missing from the flat or with the B flag, 0 or more than 8 borders, a border
 *                                given twice, for OSPFv3, among them R, without area 0 or A2, or not a B-flag router
 *                                vertex of the flat, a usable type-3 LSA of a C in A2 for a prefix of C's table it cannot
 *                                advertise.  HSPF_E_UNSUPPORTED: an NSSA, a V-flag router in A2, a B that is a router of
 *                                A2, a usable type-4 LSA of another ABR in a C's area-0 summaries, winners that do not
 *                                fit.
 *   hspf_ospfv2_third_area_cells[16]  the arguments of hspf_ospfv2_backbone_cells[16] (border_cells: each C's cells
 *                                of the job) plus border_entries (per border a device u32 [n_jobs][G_b] of its
 *                                entries, NULL allowed for a border without groups and for a table without chain
 *                                slots) and border_entry_status (per border the entries call's device u32[n_jobs]
 *                                words or NULL; the array may be NULL).  A job's status word ORs R's row-0 word, each
 *                                C's cell status and entries status; a job with a non-zero word gets empty cells.
 *                                HSPF_E_INVAL for a table that is not a third-area one.  A table without chain slots
 *                                also runs through hspf_ospfv2_backbone[_asbr]_cells[16] / _delta[16]; those refuse a
 *                                third-area table with chain slots (HSPF_E_INVAL), before any launch.  Nothing is
 *                                launched for 0 jobs.  Enqueued on the ctx stream.
 *   hspf_ospfv2_third_area_delta[16]  the route-delta stage over the same walk (base cells as hspf_ospfv2_rib_delta).
 */
int hspf_ospfv2_third_area_table_create(const hspf_ospfv2_flat *flat, uint32_t router_id,
                                        const struct hl_ospf_area_config *config,
                                        const hl_ospfv2_summary_lsa *summaries, uint32_t n_summaries,
                                        const hl_ospfv2_external_lsa *externals, uint32_t n_externals,
                                        const hspf_ospfv2_abr_backbone_table *const *borders, uint32_t n_borders,
                                        hspf_ospfv2_backbone_table **out);
int hspf_ospfv2_third_area_cells(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                 const uint32_t *const *border_entry_status, uint32_t *job_status_out,
                                 hl_ospf_rib_cell *cells);
int hspf_ospfv2_third_area_cells16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                   const uint32_t *const *border_entry_status, uint32_t *job_status_out,
                                   hl_ospf_rib_cell *cells);
int hspf_ospfv2_third_area_delta(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                 const hspf_result *planes, const hl_ospf_rib_cell *const *border_cells,
                                 const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                 const uint32_t *const *border_entry_status, const hl_ospf_rib_cell *base_cells,
                                 uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                                 hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_ospfv2_third_area_delta16(hspf_ctx *ctx, const hspf_ospfv2_backbone_table *t, uint32_t n_jobs,
                                   const hspf_result16 *planes, const hl_ospf_rib_cell *const *border_cells,
                                   const uint32_t *const *border_status, const uint32_t *const *border_entries,
                                   const uint32_t *const *border_entry_status, const hl_ospf_rib_cell *base_cells,
                                   uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                                   hl_route_delta *records, uint64_t cap, uint64_t *n_records);

/*
 * The same stage for OSPFv3.  The table is an hspf_ospfv2_backbone_table marked OSPFv3; the cells and delta calls
 * above take it (the table's mark picks the walk), and each version's create and decode refuse the other version's
 * tables (HSPF_E_INVAL).  For job j, with border b's ABR cells of j decoded to rib_b (hspf_ospfv3_abr_rib_from_cells),
 * the decoded cells of j equal the affected-prefix routes, prefix options included, of
 *     hspf_ospfv3_update_rib_full(R, max_paths, [{0, area_from_planes(area 0, R's row 0), ifaces, S_j, 1}], X)
 * where S_j is area 0's Inter-Area-Prefix / Inter-Area-Router LSAs with each border's Inter-Area-Prefix LSAs
 * replaced by hspf_ospfv3_net_summaries(rib_b, target area 0), in LsaKey order.  A border advertises a route as the
 * OSPFv2 stage says, and its LSA carries the prefix options of the border cell's winning intra-area record, as the
 * OSPFv3 intra-area decode reads them.  A slot's winner is n_records + (slot index << 8 | those options): a border
 * route that changes record at an equal metric, to one with other options, changes R's winner, and the route-delta
 * stage reports OTHER.
 *
 *   hspf_ospfv3_backbone_table_create  host.  As hspf_ospfv2_backbone_table_create, over R's OSPFv3 area-0 flat, area
 *                                0's Inter-Area-Prefix / Inter-Area-Router LSAs in LsaKey order, the AS-external LSAs
 *                                and the borders' OSPFv3 ABR tables.  Inter-Area-Prefix LSAs with the NU option are
 *                                left out, as update_rib_full leaves them out.  Refusals: those of the OSPFv2 call,
 *                                with an OSPFv2 border table HSPF_E_INVAL, a usable Inter-Area-Router LSA from a border
 *                                HSPF_E_UNSUPPORTED, and slot winners that would not fit 32 bits HSPF_E_UNSUPPORTED.
 *   hspf_ospfv3_backbone_table_prefixes6  P, and the IPv6 prefixes / lengths in prefix order (pointers may be NULL);
 *                                HSPF_E_INVAL for an OSPFv2 table.
 *   hspf_ospfv3_backbone_from_cells host: one job's cells -> the table of the contract, a slot winner's prefix options
 *                                read from the winner.  area: R's image of the table's area (area 0 here, the target
 *                                area of an hspf_ospfv3_nonbackbone_table_create table); gathers as
 *                                hspf_ospfv2_backbone_from_cells.
 */
int hspf_ospfv3_backbone_table_create(const struct hspf_ospfv3_flat *flat, uint32_t router_id,
                                      const hl_ospfv3_inter_area_lsa *summaries, uint32_t n_summaries,
                                      const hl_ospfv3_external_lsa *externals, uint32_t n_externals,
                                      const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders,
                                      hspf_ospfv2_backbone_table **out);
int hspf_ospfv3_backbone_table_prefixes6(const hspf_ospfv2_backbone_table *t, uint32_t *n_prefixes,
                                         const hl_ip_addr **prefixes, const uint32_t **lens);
int hspf_ospfv3_backbone_from_cells(const hspf_ospfv2_backbone_table *t, const hl_ospfv3_area *area,
                                    const hl_ospf_rib_cell *cells, const uint32_t *gather_v, const uint64_t *gather_nh,
                                    uint32_t n_gather, hl_ospfv3_rib *out);

/*
 * The same OSPFv3 stage with the borders' Inter-Area-Router LSAs re-originated per job: a border originates one into
 * area 0 for router A (an ASBR) when A is a router with the E flag in one of its non-backbone areas that it reaches,
 * below LSInfinity, in the job; its metric is that distance (hspf_ospfv3_rtr_summaries' rule; an id in two such areas
 * keeps the later area's).  For job j, with border b's cells decoded to rib_b over its areas areas_b, the decoded
 * cells of j equal the affected-prefix routes, prefix options included, of the hspf_ospfv3_update_rib_full above,
 * with S_j holding each border's Inter-Area-Prefix LSAs from hspf_ospfv3_net_summaries(rib_b, areas_b, target area 0)
 * AND its Inter-Area-Router LSAs from hspf_ospfv3_rtr_summaries(areas_b, target area 0), in LsaKey order.  R's entry
 * for A is the last usable Inter-Area-Router LSA, in LsaKey order, whose ABR R reaches (rib_full step 2 replaces the
 * entry per LSA), not the cheapest.  The options of an Inter-Area-Router LSA are outside the contract, as they are for
 * hspf_ospfv3_rtr_summaries.  The Inter-Area-Router rules are restated from the reference's code: no recorded
 * conformance data holds an Inter-Area-Router LSA, so their parity rests on the host restatement alone.
 *
 *   hspf_ospfv3_backbone_asbr_table_create  host.  Arguments as hspf_ospfv3_backbone_table_create; the result may hold
 *                                Inter-Area-Router slots, as hspf_ospfv2_backbone_asbr_table_create's type-4 slots:
 *                                per ASBR A some border can originate for, the static records of other ABRs and one
 *                                slot per (border, non-backbone area where A is an E-flag router) at the border's place
 *                                in LsaKey order.  The affected prefixes add every prefix of a usable AS-external LSA
 *                                of such an A.  The refusals of hspf_ospfv3_backbone_table_create apply, except the one
 *                                of a border's Inter-Area-Router LSA, and: HSPF_E_INVAL a usable Inter-Area-Router LSA
 *                                of a border for a router it cannot originate for (the NU option does not make one
 *                                unusable: NU leaves out prefixes only); HSPF_E_UNSUPPORTED a router with the E and the
 *                                B flag in a border's non-backbone area, or slots reading more than 8 (border, area)
 *                                plane sets.  The table is marked as this call's: hspf_ospfv2_backbone_table_asbr_slots
 *                                counts its slots, hspf_ospfv3_backbone_from_cells decodes it (an external cell's
 *                                winner is its AS-external record, whose prefix options the route takes), and the asbr
 *                                calls above take it.  Those calls refuse an OSPFv3 area-0 table of
 *                                hspf_ospfv3_backbone_table_create (HSPF_E_INVAL), before any launch.
 *   hspf_ospfv2_backbone_asbr_cells[16] / _delta[16]  over this table: with Inter-Area-Router slots, the walk above
 *                                with the arguments and job status rule of the OSPFv2 asbr calls; without slots, the
 *                                output of hspf_ospfv2_backbone_cells[16] / _delta[16].  The cells and delta calls
 *                                without asbr refuse a table with slots (HSPF_E_INVAL).
 */
int hspf_ospfv3_backbone_asbr_table_create(const struct hspf_ospfv3_flat *flat, uint32_t router_id,
                                           const hl_ospfv3_inter_area_lsa *summaries, uint32_t n_summaries,
                                           const hl_ospfv3_external_lsa *externals, uint32_t n_externals,
                                           const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders,
                                           hspf_ospfv2_backbone_table **out);

/*
 * Non-backbone router over what-if jobs on the backbone, OSPFv3: hspf_ospfv2_nonbackbone_table_create's stage over
 * Inter-Area-Prefix / Inter-Area-Router LSAs.  R is an internal router of a non-backbone area A, a job changes costs
 * in area 0 only, and the borders are A's ABRs attached to area 0 (every one of them must be given).  The borders'
 * cells of job j come from hspf_ospfv3_abr_rib_cells[16], with each border's area-0 row of the job and row 0 of its
 * other areas.  For job j, with border b's cells decoded to rib_b (hspf_ospfv3_abr_rib_from_cells) over its areas
 * areas_b, the decoded cells of j equal the affected-prefix routes, prefix options included, of
 *     hspf_ospfv3_update_rib_full(R, max_paths, [{A, area_from_planes(A, R's row 0), ifaces, S_j, 1}], X)
 * where S_j is A's Inter-Area-Prefix / Inter-Area-Router LSAs with each border's LSAs replaced by
 * hspf_ospfv3_net_summaries(rib_b, areas_b, target A) and hspf_ospfv3_rtr_summaries(areas_b, target A), both over
 * the border's area-0 SPF of the job, in LsaKey order.  A border advertises a route of its cell as the OSPFv2 stage
 * says (intra-area or inter-area), and its LSA carries the route's prefix options: those of the winning intra-area
 * record, or of the winning Inter-Area-Prefix record of an inter-area cell (a transit-area record included).  A
 * slot's winner is n_records + (slot index << 8 | those options), so a border route whose winning LSA changes at an
 * equal metric, to one with other options, shows as OTHER in the route-delta stage.  Inter-Area-Router slots are the
 * OSPFv2 stage's type-4 slots: one per (border, area other than A where the ASBR is an E-flag router), an area-0
 * ASBR's read from the border's area-0 row of the job.  The affected prefixes and the stub-area rules are those of
 * the OSPFv2 stage, the stub default route being ::/0.
 *
 *   hspf_ospfv3_nonbackbone_table_create  host.  flat: R's OSPFv3 area-A flat (A is flat's area id); config: A's
 *                                configuration; summaries: A's Inter-Area-Prefix / Inter-Area-Router LSAs in LsaKey
 *                                order; externals: the AS-external LSAs; borders: the borders' OSPFv3 ABR tables.  The
 *                                result is an hspf_ospfv2_backbone_table marked OSPFv3 and with its target area A; the
 *                                cells and delta calls of both kinds take it (a table with Inter-Area-Router slots is
 *                                the asbr calls', as for OSPFv2), and hspf_ospfv3_backbone_from_cells decodes it over
 *                                R's image of A.  Refusals:
 *                                those of hspf_ospfv2_nonbackbone_table_create, over Inter-Area-Prefix /
 *                                Inter-Area-Router LSAs, with an OSPFv2 border table HSPF_E_INVAL and slot winners that
 *                                would not fit 32 bits HSPF_E_UNSUPPORTED.  Inter-Area-Prefix LSAs with the NU option
 *                                are left out.
 */
int hspf_ospfv3_nonbackbone_table_create(const struct hspf_ospfv3_flat *flat, uint32_t router_id,
                                         const struct hl_ospf_area_config *config,
                                         const hl_ospfv3_inter_area_lsa *summaries, uint32_t n_summaries,
                                         const hl_ospfv3_external_lsa *externals, uint32_t n_externals,
                                         const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders,
                                         hspf_ospfv2_backbone_table **out);

/*
 * Non-backbone router over what-if jobs inside another non-backbone area, OSPFv3: the
 * hspf_ospfv2_third_area_table_create stage over Inter-Area-Prefix / Inter-Area-Router LSAs, with the same contract on
 * jobs, borders (the C's, each an hspf_ospfv3_abr_backbone_table_create table over A1's ABRs) and affected prefixes.
 * For job j, with C's cells of j (hspf_ospfv2_abr_backbone_cells[16] over its OSPFv3 table) decoded to rib_C
 * (hspf_ospfv3_abr_backbone_from_cells), the decoded cells of j equal the affected-prefix routes, prefix options
 * included, of
 *     hspf_ospfv3_update_rib_full(R, max_paths, [{A2, area_from_planes(A2, R's row 0), ifaces, S_j, 1}], X)
 * where S_j is A2's Inter-Area-Prefix / Inter-Area-Router LSAs with each C's replaced by
 * hspf_ospfv3_net_summaries(rib_C, areas_C, target A2) and hspf_ospfv3_rtr_summaries(areas_C, target A2), in LsaKey
 * order; that is the three-step host chain: each B's update_rib_full, net and rtr summaries into area 0 spliced into
 * C's area 0; each C's same chain over those LSAs into A2; update_rib_full at R.  A C's Inter-Area-Prefix LSA carries
 * the prefix options of C's route: those of its winning intra-area record or Inter-Area-Prefix record, and for a route
 * through a B's slot those the B copied from its own route, which C's cell winner carries (n_recs_C + (slot << 8 |
 * options)).  R's slot winner is n_records + (slot index << 8 | those options), so a B route that changes record at an
 * equal metric, to one with other options, changes R's winner through C, and the route-delta stage reports OTHER.  When
 * A1 holds an ASBR A, each C's Inter-Area-Router LSA for A into a normal A2 is a chain slot, as for OSPFv2, reading C's
 * entries of the job (hspf_ospfv3_abr_backbone_asbr_entries[16]).  The options of an Inter-Area-Router LSA are outside
 * the contract, as they are for hspf_ospfv3_rtr_summaries.
 *
 *   hspf_ospfv3_third_area_table_create  host.  The arguments of hspf_ospfv2_third_area_table_create over OSPFv3: R's
 *                                area-A2 flat, A2's configuration, A2's Inter-Area-Prefix / Inter-Area-Router LSAs in
 *                                LsaKey order, the AS-external LSAs, and the C's OSPFv3 abr_backbone tables, which must
 *                                outlive the table.  The result is an hspf_ospfv2_backbone_table marked OSPFv3 and as a
 *                                third-area table: hspf_ospfv2_backbone_table_* (asbr_slots: the chain slot count and 0
 *                                plane sets), _upload, hspf_ospfv3_backbone_table_prefixes6 and
 *                                hspf_ospfv3_backbone_from_cells take it (an external route reached through a chain
 *                                slot decodes as any external route).  Refusals: those of the OSPFv2 call, with an
 *                                OSPFv2 border table HSPF_E_INVAL (and the OSPFv2 call refuses an OSPFv3 one) and slot
 *                                winners that would not fit 32 bits (n_records + (slots << 8)) HSPF_E_UNSUPPORTED.
 *                                Inter-Area-Prefix LSAs with the NU option are left out.
 *   hspf_ospfv2_third_area_cells[16] / _delta[16]  take it; its version mark picks the walk, which reads C's slot
 *                                winners, with or without chain slots.  The status-word rule is the OSPFv2 one: a job's
 *                                word ORs R's row-0 word, each C's cell status and entries status, and a job with a
 *                                non-zero word gets empty cells.  hspf_ospfv2_backbone[_asbr]_cells[16] / _delta[16]
 *                                refuse an OSPFv3 third-area table, with or without chain slots (HSPF_E_INVAL), before
 *                                any launch: their walks cannot read C's slot winners.
 *   hspf_ospfv3_abr_backbone_asbr_entries[16]  hspf_ospfv2_abr_backbone_asbr_entries[16] over an OSPFv3 C table (the
 *                                Inter-Area-Router rows of hspf_ospfv3_rtr_summaries(areas_C, target a normal area
 *                                other than area 0) over C's areas of the job); hspf_ospfv2_abr_backbone_table_asbrs
 *                                names its groups.  HSPF_E_INVAL: an OSPFv2 table, and the OSPFv2 call's refusals.
 */
int hspf_ospfv3_third_area_table_create(const struct hspf_ospfv3_flat *flat, uint32_t router_id,
                                        const struct hl_ospf_area_config *config,
                                        const hl_ospfv3_inter_area_lsa *summaries, uint32_t n_summaries,
                                        const hl_ospfv3_external_lsa *externals, uint32_t n_externals,
                                        const hspf_ospfv2_abr_backbone_table *const *borders, uint32_t n_borders,
                                        hspf_ospfv2_backbone_table **out);
int hspf_ospfv3_abr_backbone_asbr_entries(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                          const hspf_result *planes, const hspf_result *const *border_planes,
                                          const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                          uint32_t *job_status_out, uint32_t *entries);
int hspf_ospfv3_abr_backbone_asbr_entries16(hspf_ctx *ctx, const hspf_ospfv2_abr_backbone_table *t, uint32_t n_jobs,
                                            const hspf_result16 *planes, const hspf_result16 *const *border_planes,
                                            const uint32_t *const *border_n_rows, const uint32_t *const *border_rows,
                                            uint32_t *job_status_out, uint32_t *entries);

/*
 * Area border router over what-if jobs inside an area it is not attached to, OSPFv3: the
 * hspf_ospfv2_abr_backbone_table_create stage over Inter-Area-Prefix / Inter-Area-Router LSAs, with the same
 * contract on jobs and borders.  The borders' cells of job j come from hspf_ospfv2_abr_rib_cells[16] over their
 * hspf_ospfv3_abr_ribtable_create tables, with each border's row of the perturbed area for the job and row 0 of its
 * other areas.  For job j, with border b's cells of j decoded to rib_b (hspf_ospfv3_abr_rib_from_cells) over its areas
 * areas_b, the decoded cells of j equal the affected-prefix routes, prefix options included, of
 *     hspf_ospfv3_update_rib_full(R, max_paths, [{A_i.area_id, area_from_planes(A_i, R's row 0 of A_i), ifaces,
 *         S_i, active_i}], X)
 * where S_i is area i's Inter-Area-Prefix / Inter-Area-Router LSAs, area 0's with each border's own replaced by
 * hspf_ospfv3_net_summaries(rib_b, areas_b, target area 0) and hspf_ospfv3_rtr_summaries(areas_b, target area 0), in
 * LsaKey order.  A border advertises a route as the OSPFv2 stage says, and its LSA carries the prefix options of the
 * border cell's winning intra-area record; the Inter-Area-Router slots are the OSPFv2 stage's type-4 slots.  The
 * options of an Inter-Area-Router LSA are outside the contract, as they are for hspf_ospfv3_rtr_summaries.
 *
 *   hspf_ospfv3_abr_backbone_table_create  host.  The arguments of hspf_ospfv3_abr_ribtable_create (R's OSPFv3 areas in
 *                                instance order; area 0's LSAs as in R's LSDB, borders' LSAs included), plus the
 *                                borders' OSPFv3 ABR tables, which must outlive the table.  The result is an
 *                                hspf_ospfv2_abr_backbone_table marked OSPFv3: hspf_ospfv2_abr_backbone_table_free /
 *                                _records / _upload and hspf_ospfv2_abr_backbone_cells[16] / _delta[16] take it (the
 *                                mark picks the walk), and a slot's winner is n_records + (slot index << 8 | the prefix
 *                                options of the border's LSA): a border route that changes record at an equal metric,
 *                                to one with other options, changes R's winner, and the route-delta stage reports
 *                                OTHER.  Refusals: those of the OSPFv2 call, with an OSPFv2 border table HSPF_E_INVAL
 *                                and slot winners that would not fit 32 bits HSPF_E_UNSUPPORTED.  Inter-Area-Prefix
 *                                LSAs with the NU option are left out, a border's included.
 *   hspf_ospfv3_abr_backbone_table_prefixes6  P, and the IPv6 prefixes / lengths in prefix order (pointers may be
 *                                NULL); HSPF_E_INVAL for an OSPFv2 table.
 *   hspf_ospfv3_abr_backbone_from_cells  host: one job's cells -> exactly the routes of the affected prefixes of the
 *                                contract, a slot winner's prefix options read from the winner.  areas: R's
 *                                hl_ospfv3_area images in the table's order; gathers as
 *                                hspf_ospfv2_abr_backbone_from_cells.  The create and decode of each version refuse a
 *                                table of the other (HSPF_E_INVAL).
 */
int hspf_ospfv3_abr_backbone_table_create(uint32_t router_id, uint32_t n_areas, const struct hspf_ospfv3_flat *const *flats,
                                          const uint32_t *area_ids, const hl_ospfv3_inter_area_lsa *const *summaries,
                                          const uint32_t *n_summaries, const uint8_t *active,
                                          const hl_ospfv3_external_lsa *externals, uint32_t n_externals,
                                          const hspf_ospfv2_abr_ribtable *const *borders, uint32_t n_borders,
                                          hspf_ospfv2_abr_backbone_table **out);
int hspf_ospfv3_abr_backbone_table_prefixes6(const hspf_ospfv2_abr_backbone_table *t, uint32_t *n_prefixes,
                                             const hl_ip_addr **prefixes, const uint32_t **lens);
int hspf_ospfv3_abr_backbone_from_cells(const hspf_ospfv2_abr_backbone_table *t, const hl_ospfv3_area *areas,
                                        uint32_t n_areas, const hl_ospf_rib_cell *cells, const uint32_t *gather_area,
                                        const uint32_t *gather_v, const uint64_t *gather_nh, uint32_t n_gather,
                                        hl_ospfv3_rib *out);

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
 * Summary-LSA origination of an area border router (compute_net_summaries / compute_rtr_summaries,
 * holo-ospf/src/area.rs:561-740), for one target area, over the table update_rib_full left:
 *   rib       hspf_ospfv2_update_rib_full's output;  rtrs  hspf_ospfv2_rib_router_tables' output (same inputs);
 *   areas     the router's areas as given to those calls (area_id, ifaces, active are read);
 *   config    per area: its type, whether it takes regular summaries, the cost of its default route.
 * out[0, *n_out): the type-3 contents (lsa_type 3, lsa_id = the prefix address, mask, metric) in prefix order, then the
 * type-4 contents (lsa_type 4, lsa_id = the ASBR's router id, mask 0, metric) in router-id order; adv_rtr = router_id.
 * Nothing when at most one area is active (not an ABR).  Type 3: every intra- or inter-area route below LSInfinity
 * that is not of the target area, only intra-area ones into the backbone, none with a next hop on one of the target
 * area's interfaces; in a stub or NSSA area, the default route at default_cost (and, with summary = 0, nothing else).
 * Type 4: into a normal area, each other area's router entry with the E flag below LSInfinity, intra-area ones only
 * into the backbone, under the same next-hop rule; an id in two areas keeps the later area's.  Out of the contract:
 * LSA ids (the reference keeps them across runs), and area ranges (no range may be configured).  HSPF_E_NOMEM with
 * *n_out set when cap is too small.  Host only.
 */
#define HL_AREA_NORMAL 0u
#define HL_AREA_STUB   1u
#define HL_AREA_NSSA   2u
typedef struct hl_ospf_area_config {
    uint32_t default_cost;     /* area.config.default_cost (10 by default)                */
    uint8_t  area_type;        /* HL_AREA_*                                               */
    uint8_t  summary;          /* area.config.summary (1 by default; 0: totally stubby)   */
    uint8_t  _pad[2];
} hl_ospf_area_config;
int hspf_ospfv2_net_summaries(uint32_t router_id, const hl_ospfv2_rib *rib, const hl_ospfv2_rtr_tables *rtrs,
                              const hl_ospfv2_rib_area *areas, const hl_ospf_area_config *config, uint32_t n_areas,
                              uint32_t target, hl_ospfv2_summary_lsa *out, uint32_t cap, uint32_t *n_out);
/*
 * The Inter-Area-Prefix contents an OSPFv3 area border router originates into one target area (compute_net_summaries,
 * lsa_orig_inter_area_network of holo-ospf ospfv3/lsdb.rs:341-386), over hspf_ospfv3_update_rib_full's table: the
 * type-3 rules of hspf_ospfv2_net_summaries, each LSA carrying its route's prefix options (the default route of a stub
 * area: ::/0 at default_cost, options 0).  out[0, *n_out): lsa_type 3, adv_rtr = router_id, lsa_id 0, the prefix, its
 * length, prefix options and metric, in prefix order.  Inter-Area-Router contents: hspf_ospfv3_rtr_summaries.
 * HSPF_E_NOMEM with *n_out set when cap is too small.  Host only.
 */
int hspf_ospfv3_net_summaries(uint32_t router_id, const hl_ospfv3_rib *rib, const hl_ospfv3_rib_area *areas,
                              const hl_ospf_area_config *config, uint32_t n_areas, uint32_t target,
                              hl_ospfv3_inter_area_lsa *out, uint32_t cap, uint32_t *n_out);
/*
 * The Inter-Area-Router contents an OSPFv3 area border router originates into one target area (compute_rtr_summaries,
 * holo-ospf area.rs:699-740), over the router entries hspf_ospfv3_update_rib_full leaves for the same `areas` (each
 * area's SPF routers as intra-area entries, then inter-area entries from the Inter-Area-Router LSAs it reads: area 0's
 * when more than one area is active).  The type-4 rule of hspf_ospfv2_net_summaries: only into a normal area, each
 * entry of another area with the E flag below LSInfinity, intra-area ones only into the backbone, none with a next
 * hop on one of the target area's interfaces, an id in two areas keeping the later area's entry.  out[0, *n_out):
 * lsa_type 4, adv_rtr = router_id, router_id = the ASBR, metric, lsa_id 0, in router-id order.  Nothing when at most
 * one area is active.  The LSA's options are out of the contract: hl_ospfv3_inter_area_lsa has no field for them,
 * and update_rib_full does not read them.  HSPF_E_NOMEM with *n_out set when cap is too small.  Host only.
 */
int hspf_ospfv3_rtr_summaries(uint32_t router_id, const hl_ospfv3_rib_area *areas, const hl_ospf_area_config *config,
                              uint32_t n_areas, uint32_t target, hl_ospfv3_inter_area_lsa *out, uint32_t cap,
                              uint32_t *n_out);

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
/* The batched routing-table stage for OSPFv3 areas (see "Batched routing-table stage" above): for job j with root
 * router r over area A, the decoded cells of j equal
 *     hspf_ospfv3_update_rib_full(r, A.max_paths, [{A.area_id, spf_j, A.ifaces, summaries, active = 1}], externals)
 * with spf_j = hspf_ospfv3_area_from_planes(A with router_id = r, j's planes): routes (prefix options, tag, type-2
 * metric, area) and next hops.
 *   hspf_ospfv3_ribtable_create   the same hspf_ospfv2_ribtable: the intra-area records of hspf_ospfv3_rtable_create,
 *                                 then the type-3 / type-5 / ASBR-slot / type-4 records, as hspf_ospfv2_ribtable_create
 *                                 builds them, with the rules of hspf_ospfv3_update_rib_full: an Inter-Area-Prefix or
 *                                 AS-external LSA with the NU option is left out, an Inter-Area-Router LSA names its
 *                                 ASBR in router_id, and prefixes are ordered by their 16 address bytes, then length.
 *                                 summaries: the area's Inter-Area-Prefix / Inter-Area-Router LSAs (LsaKey order);
 *                                 externals: the instance's AS-external LSAs.  A router vertex's flags are those of its
 *                                 first Router-LSA fragment.  The same two HSPF_E_UNSUPPORTED refusals as OSPFv2.
 *                                 hspf_ospfv2_ribtable_free / _prefixes / _contributors / _arrays (prefix[] all zero) /
 *                                 _upload and hspf_ospfv2_rib_cells[16] / hspf_ospfv2_rib_delta[16] take it unchanged.
 *   hspf_ospfv3_ribtable_prefixes6  the table's prefixes (IPv6 networks, as update_rib_full names them) and lengths.
 *   hspf_ospfv3_rib_from_cells    host: one job's cells -> the table above, as hspf_ospfv2_rib_from_cells (next hops
 *                                 named by interface sort key in NexthopKey order, HSPF_E_NOMEM with the counts,
 *                                 HSPF_E_UNSUPPORTED in the cases of hspf_ospfv3_routes_from_cells).  HSPF_E_INVAL for
 *                                 an OSPFv2 table, as hspf_ospfv2_rib_from_cells gives for an OSPFv3 one. */
int hspf_ospfv3_ribtable_create(const hspf_ospfv3_flat *flat, uint32_t area_id, const hl_ospfv3_inter_area_lsa *summaries,
                                uint32_t n_summaries, const hl_ospfv3_external_lsa *externals, uint32_t n_externals,
                                hspf_ospfv2_ribtable **out);
int hspf_ospfv3_ribtable_prefixes6(const hspf_ospfv2_ribtable *rt, const hl_ip_addr **prefixes, const uint32_t **lens);
int hspf_ospfv3_rib_from_cells(const hl_ospfv3_area *area, const hspf_ospfv2_ribtable *rt, const hl_ospf_rib_cell *cells,
                               const uint32_t *gather_v, const uint64_t *gather_nh, uint32_t n_gather, hl_ospfv3_rib *out);
/* The batched routing-table stage for OSPFv3 area border routers (see "Batched routing-table stage on the device for
 * one area border router" above): with attached areas A_0 .. A_{n-1} (flat, area id, Inter-Area-Prefix /
 * Inter-Area-Router LSAs in LsaKey order, active) and AS-external LSAs X, the decoded cells of job j equal
 *     hspf_ospfv3_update_rib_full(r, max_paths,
 *         [{A_i.area_id, hspf_ospfv3_area_from_planes(A_i, planes_i[rows[j][i]]), A_i.ifaces, summaries_i, active_i}],
 *         X)
 * routes (prefix options, tag, type-2 metric, area) and next hops, the areas in the caller's order.
 *   hspf_ospfv3_abr_ribtable_create  the same hspf_ospfv2_abr_ribtable, built as hspf_ospfv2_abr_ribtable_create builds
 *                                 it (same arguments per area, same refusals) over each area's
 *                                 hspf_ospfv3_ribtable_create table, with that call's OSPFv3 rules (NU-option LSAs left
 *                                 out, an Inter-Area-Router LSA names its ASBR in router_id, IPv6 prefix order).  An
 *                                 area 0 with V-flag routers is accepted here: the walk's transit-area step covers it.
 *                                 The table carries its prefixes as IPv6 networks and the prefix options of every
 *                                 Inter-Area-Prefix and AS-external record.  hspf_ospfv2_abr_ribtable_free / _prefixes /
 *                                 _contributors / _arrays (prefix[] all zero) / _areas / _upload and
 *                                 hspf_ospfv2_abr_rib_cells[16] / hspf_ospfv2_abr_rib_delta[16] take it unchanged.
 *   hspf_ospfv3_abr_ribtable_prefixes6  the table's prefixes and lengths; HSPF_E_INVAL for an OSPFv2 table.
 *   hspf_ospfv3_abr_rib_from_cells  host: one job's cells -> the table above, as hspf_ospfv2_abr_rib_from_cells (areas:
 *                                 each area's image with router_id = the router, in the table's order).  When
 *                                 intra-area routes of two areas tie, the route keeps the prefix options of the first
 *                                 area in that order, as update_rib_full keeps the first route it met.  HSPF_E_INVAL
 *                                 for an OSPFv2 table, as hspf_ospfv2_abr_rib_from_cells gives for an OSPFv3 one. */
int hspf_ospfv3_abr_ribtable_create(uint32_t router_id, uint32_t n_areas, const hspf_ospfv3_flat *const *flats,
                                    const uint32_t *area_ids, const hl_ospfv3_inter_area_lsa *const *summaries,
                                    const uint32_t *n_summaries, const uint8_t *active,
                                    const hl_ospfv3_external_lsa *externals, uint32_t n_externals,
                                    hspf_ospfv2_abr_ribtable **out);
int hspf_ospfv3_abr_ribtable_prefixes6(const hspf_ospfv2_abr_ribtable *t, const hl_ip_addr **prefixes,
                                       const uint32_t **lens);
int hspf_ospfv3_abr_rib_from_cells(const hspf_ospfv2_abr_ribtable *t, const hl_ospfv3_area *areas, uint32_t n_areas,
                                   const hl_ospf_rib_cell *cells, const uint32_t *gather_area, const uint32_t *gather_v,
                                   const uint64_t *gather_nh, uint32_t n_gather, hl_ospfv3_rib *out);
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
 * Routing table of an IS-IS L1/L2 router on the device, for every job of a what-if batch: update_rib
 * (holo-isis/src/route.rs:182-249) over the job's SPTs of both levels.  The L1 table, the active summaries it
 * gives (get_spm: the SHORTEST configured match of each L1 route; metric: the configured one, else the lowest
 * covered L1 metric), the L2 table in which an active summary replaces the route of its prefix with a blackhole
 * route, and the two merged with the L1 route preferred (isis_l1l2_rib_cells.h).
 *
 *   hspf_isis_l1l2_ribtable_create   per L1/L2 router: `l1` / `l2` its instance images of level 1 and 2 (level_type 3,
 *                             the same system id and max_paths), `cfg` its n_cfg configured summaries in prefix order
 *                             (IPv4 before IPv6, address, length).  Each level's contributors are those of
 *                             hspf_isis_rtable_create.  The prefixes are the union of both levels' prefixes and the
 *                             summary prefixes, in hl_isis_rib order; per prefix an L1 range, an L2 range and its
 *                             summary.  Contributor indices (hl_isis_route_cell.winner) share one space: the L1
 *                             contributors, the L2 contributors, then one index per configured summary.
 *     l2_derived              one byte per entry of l2->lvl.ipreaches (NULL: none): non-zero marks an entry of the
 *                             router's own (non-pseudonode) L2 LSPs that is not configured there — lsp_propagate_l1_to_l2 or an
 *                             advertised summary put it there.  Those entries are left out of the L2 contributors.
 *                             The L2 LSDB holds the base state's propagation; in a what-if job holo re-originates
 *                             that LSP from the job's L1 SPT, and a stale entry would become a connected L2 route
 *                             holo does not have.  Leaving them out is exact: whenever the re-originated LSP
 *                             carries a propagated entry, its originator is on the job's L1 SPT of the same
 *                             topology, so the prefix has an L1 route, and the L1 route wins the merge; an active
 *                             summary replaces the L2 route of its prefix anyway.  That holds when every L1 entry
 *                             propagation's static filters let through (holo-isis lsdb.rs:1163-1258) is one
 *                             compute_routes feeds into the L1 table (spf.rs:862-882, 1141): the builder checks
 *                             it and returns HSPF_E_UNSUPPORTED for a fragment whose system has no valid zeroth
 *                             LSP, an extended IPv4 entry above the wide-metric limit, or an MT-IPv6 entry under
 *                             an instance with IPv6 disabled, unless a summary covers it.  What-if jobs change
 *                             costs only, so the check is exact for every job.
 *                             HSPF_E_INVAL: levels or level types wrong, system ids or max_paths differ, `cfg` out
 *                             of order, a non-zero l2_derived byte for an entry outside the router's own
 *                             (non-pseudonode) L2 LSPs.
 *   hspf_isis_l1l2_ribtable_topology vertex count and root vertex of level 1 or 2, topology 0 or 1 (as
 *                             hspf_isis_rtable_topology).
 *   hspf_isis_l1l2_ribtable_arrays   prefix[P], len[P], off (u32: the L1 ranges [P + 1], the L2 ranges [P + 1], ...),
 *                             contribs (the L1 then the L2 contributor records); any pointer may be NULL.
 *   hspf_isis_l1l2_ribtable_summaries n_l1 (the number of L1 contributors), S, sum_of[P] (0xFFFFFFFF: not a summary
 *                             prefix), cov_off[S + 1] and cov: the L1 prefixes each summary is the shortest match of.
 *   hspf_isis_l1l2_ribtable_upload   copies the table to the ctx's device.
 *   hspf_isis_l1l2_rib_cells[16]   DEVICE planes of four topologies: l1_std, l1_mt6 from one L1 batch and l2_std,
 *                             l2_mt6 from one L2 batch (hspf_run_batch_async / hspf_run_batch16_async, the wide ones
 *                             with nh_words == 1; *_mt6 may be NULL unless that level's table has an MT-IPv6 root).
 *                             n_rows[2]: the rows of the L1 and of the L2 batch; rows [n_jobs][2] (device): the
 *                             job's L1 row and L2 row, so that a job perturbing one level reuses the other level's
 *                             plain row.  First the summary pass, one warp per (job, summary), writes
 *                             summary_out (device u64 [n_jobs][S], required when S > 0): 0 inactive,
 *                             (1 << 32) | lowest covered L1 metric when active — per job, which summaries the router
 *                             advertises into L2 and at what metric.  Then cells[n_jobs][P] (device).
 *                             job_status_out (device [n_jobs], or NULL): the OR of the status words of the job's
 *                             rows (MT-IPv6 planes only where the level has an MT-IPv6 root), HSPF_JS_INVALID for a
 *                             row out of range.  A job with a non-zero status gets empty cells and summary words 0.
 *                             Nothing is launched for 0 jobs.  Enqueued on the ctx stream; no synchronisation.
 *   hspf_isis_l1l2_rib_delta[16]   the summary pass, then the route-delta stage (below) over the same walk.
 *   hspf_isis_l1l2_rib_from_cells  host: one job's cells and summary words -> exactly the hl_isis_rib of
 *                             hspf_isis_rib_merge(hspf_isis_rib_add_summaries(L2 routes, hspf_isis_summaries(L1
 *                             routes, cfg)), L1 routes), the routes of each level as hspf_isis_routes_from_planes
 *                             gives them over the same planes (the L2 LSDB without the derived entries).
 *                             planes[4]: the job's planes and overrides of L1 std, L1 MT-IPv6, L2 std, L2 MT-IPv6.
 *                             HSPF_E_UNSUPPORTED as hspf_isis_routes_from_cells.
 */
typedef struct hspf_isis_l1l2_ribtable hspf_isis_l1l2_ribtable;
/* One topology's planes of one job for the host decode: dist / hops [V], its n_ov edge overrides */
typedef struct hspf_isis_job_planes {
    const uint32_t *dist;
    const uint16_t *hops;
    uint32_t n_ov;
    const uint32_t *ov_edge;
    const uint32_t *ov_cost;
} hspf_isis_job_planes;
int hspf_isis_l1l2_ribtable_create(const hl_isis_instance *l1, const hl_isis_instance *l2, const uint8_t *l2_derived,
                                   const hl_isis_summary *cfg, uint32_t n_cfg, hspf_isis_l1l2_ribtable **out);
void hspf_isis_l1l2_ribtable_free(hspf_isis_l1l2_ribtable *t);
uint32_t hspf_isis_l1l2_ribtable_prefixes(const hspf_isis_l1l2_ribtable *t);
uint32_t hspf_isis_l1l2_ribtable_contributors(const hspf_isis_l1l2_ribtable *t);
int hspf_isis_l1l2_ribtable_topology(const hspf_isis_l1l2_ribtable *t, uint32_t level, uint32_t topology,
                                     uint32_t *n_vertices, uint32_t *root);
int hspf_isis_l1l2_ribtable_arrays(const hspf_isis_l1l2_ribtable *t, const hl_ip_addr **prefix, const uint32_t **len,
                                   const uint32_t **off, const void **contribs);
int hspf_isis_l1l2_ribtable_summaries(const hspf_isis_l1l2_ribtable *t, uint32_t *n_l1, uint32_t *n_summaries,
                                      const uint32_t **sum_of, const uint32_t **cov_off, const uint32_t **cov);
int hspf_isis_l1l2_ribtable_upload(hspf_ctx *ctx, hspf_isis_l1l2_ribtable *t);
int hspf_isis_l1l2_rib_cells(hspf_ctx *ctx, const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs, const hspf_result *l1_std,
                             const hspf_result *l1_mt6, const hspf_result *l2_std, const hspf_result *l2_mt6,
                             const uint32_t *n_rows, const uint32_t *rows, uint64_t *summary_out,
                             uint32_t *job_status_out, hl_isis_route_cell *cells);
int hspf_isis_l1l2_rib_cells16(hspf_ctx *ctx, const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs,
                               const hspf_result16 *l1_std, const hspf_result16 *l1_mt6, const hspf_result16 *l2_std,
                               const hspf_result16 *l2_mt6, const uint32_t *n_rows, const uint32_t *rows,
                               uint64_t *summary_out, uint32_t *job_status_out, hl_isis_route_cell *cells);
int hspf_isis_l1l2_rib_delta(hspf_ctx *ctx, const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs, const hspf_result *l1_std,
                             const hspf_result *l1_mt6, const hspf_result *l2_std, const hspf_result *l2_mt6,
                             const uint32_t *n_rows, const uint32_t *rows, uint64_t *summary_out,
                             const hl_isis_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                             hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_isis_l1l2_rib_delta16(hspf_ctx *ctx, const hspf_isis_l1l2_ribtable *t, uint32_t n_jobs,
                               const hspf_result16 *l1_std, const hspf_result16 *l1_mt6, const hspf_result16 *l2_std,
                               const hspf_result16 *l2_mt6, const uint32_t *n_rows, const uint32_t *rows,
                               uint64_t *summary_out, const hl_isis_route_cell *base_cells, uint32_t n_base,
                               const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records,
                               uint64_t cap, uint64_t *n_records);
int hspf_isis_l1l2_rib_from_cells(const hl_isis_instance *l1, const hl_isis_instance *l2,
                                  const hspf_isis_l1l2_ribtable *t, const hl_isis_route_cell *cells,
                                  const uint64_t *summary_words, const hspf_isis_job_planes *planes, hl_isis_rib *out);

/*
 * L1 -> L2 propagation of an IS-IS L1/L2 router on the device, for every job of a what-if batch: the IP reachability
 * lsp_propagate_l1_to_l2 (holo-isis lsdb.rs:1149-1357) puts into the router's L2 LSP over the job's L1 SPT — what
 * every other L2 router of the domain sees of the area (isis_l1_to_l2_cells.h).  It tells whether an L1 failure
 * stays inside the area (absorbed by a summary, or leaving the metrics unchanged) or reaches every backbone router.
 *
 *   hspf_isis_l1_to_l2_table_create  per L1/L2 router: `l1` / `l2` its instance images of level 1 and 2, `up_down`
 *                             one byte per entry of l1->lvl.ipreaches (NULL: none set; as hspf_isis_l1_to_l2), `rib`
 *                             the router's hspf_isis_l1l2_ribtable, which supplies the configured summaries and the
 *                             summary pass; it must outlive the table and be uploaded before the device calls.  The
 *                             keys are (kind, prefix) in hspf_isis_l1_to_l2's output order: every key an entry could
 *                             be propagated into in some job, and the summary keys (IPv4: narrow and/or extended,
 *                             after the L2 metric type; IPv6).  Each propagated key keeps its records in the host
 *                             loop's order (LSP order, then entry order): the originator's L1 vertex, the entry
 *                             metric, narrow or not.  Propagation's static filters (valid non-pseudonode LSPs other
 *                             than the router's own, kinds enabled by the address families and both metric types,
 *                             MT-IPv6, up/down bits, no covering summary) hold for every job, since what-if jobs
 *                             change costs only; per job a record only asks whether its originator is reached.
 *                             HSPF_E_INVAL: levels or level types wrong, system ids differ, an l1 whose L1 vertex
 *                             counts or roots differ from the rib table's.
 *   hspf_isis_l1_to_l2_table_keys    K, the number of records, kind[K], prefix[K], len[K]; any pointer may be NULL.
 *   hspf_isis_l1_to_l2_table_upload  copies the table to the ctx's device.
 *   hspf_isis_l1_to_l2_cells[16]  DEVICE planes of the L1 batch (l1_std; l1_mt6 may be NULL unless L1 has an MT-IPv6
 *                             root; the wide ones with nh_words == 1), n_l1_rows its rows, rows [n_jobs] (device) the
 *                             job's L1 row.  L2 planes are not read.  First the summary pass of
 *                             hspf_isis_l1l2_rib_cells writes summary_out (device u64 [n_jobs][S], required when
 *                             S > 0); then cells[n_jobs][K] (device), hl_isis_route_cell: nh_mask 0, winner the
 *                             record (summary s: n_records + s), metric the advertised one (narrow totals capped at
 *                             63, wide ones at 2^32 - 1; an active summary's configured metric, else its lowest
 *                             covered L1 metric, capped at 63 for the narrow key), HL_CELL_PRESENT.  On equal totals
 *                             the first record in LSP order wins.  job_status_out (device [n_jobs], or NULL): the OR
 *                             of the job's L1 row status words, HSPF_JS_INVALID for a row out of range; such a job
 *                             gets empty cells and summary words 0.  Nothing is launched for 0 jobs.  Enqueued on the
 *                             ctx stream; no synchronisation.
 *   hspf_isis_l1_to_l2_delta[16]  the summary pass, then the route-delta stage (below) over the same walk: LOST (an
 *                             originator cut off, a summary gone inactive), GAINED, METRIC (the advertised metric),
 *                             OTHER (another originator at the same metric: the Prefix-SID may change); never NEXTHOPS.
 *   hspf_isis_l1_to_l2_from_cells  host: one job's cells and summary words -> exactly the hl_isis_ipreach list of
 *                             hspf_isis_l1_to_l2 over the job's L1 SPTs (hspf_isis_spt_from_planes of the same planes)
 *                             and the job's active summaries.  *n_out is set; HSPF_E_NOMEM when it exceeds cap.
 */
typedef struct hspf_isis_l1_to_l2_table hspf_isis_l1_to_l2_table;
int hspf_isis_l1_to_l2_table_create(const hl_isis_instance *l1, const hl_isis_instance *l2, const uint8_t *up_down,
                                    const hspf_isis_l1l2_ribtable *rib, hspf_isis_l1_to_l2_table **out);
void hspf_isis_l1_to_l2_table_free(hspf_isis_l1_to_l2_table *t);
int hspf_isis_l1_to_l2_table_keys(const hspf_isis_l1_to_l2_table *t, uint32_t *n_keys, uint32_t *n_records,
                                  const uint8_t **kind, const hl_ip_addr **prefix, const uint8_t **len);
int hspf_isis_l1_to_l2_table_upload(hspf_ctx *ctx, hspf_isis_l1_to_l2_table *t);
int hspf_isis_l1_to_l2_cells(hspf_ctx *ctx, const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs,
                             const hspf_result *l1_std, const hspf_result *l1_mt6, uint32_t n_l1_rows,
                             const uint32_t *rows, uint64_t *summary_out, uint32_t *job_status_out,
                             hl_isis_route_cell *cells);
int hspf_isis_l1_to_l2_cells16(hspf_ctx *ctx, const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs,
                               const hspf_result16 *l1_std, const hspf_result16 *l1_mt6, uint32_t n_l1_rows,
                               const uint32_t *rows, uint64_t *summary_out, uint32_t *job_status_out,
                               hl_isis_route_cell *cells);
int hspf_isis_l1_to_l2_delta(hspf_ctx *ctx, const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs,
                             const hspf_result *l1_std, const hspf_result *l1_mt6, uint32_t n_l1_rows,
                             const uint32_t *rows, uint64_t *summary_out, const hl_isis_route_cell *base_cells,
                             uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                             hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_isis_l1_to_l2_delta16(hspf_ctx *ctx, const hspf_isis_l1_to_l2_table *t, uint32_t n_jobs,
                               const hspf_result16 *l1_std, const hspf_result16 *l1_mt6, uint32_t n_l1_rows,
                               const uint32_t *rows, uint64_t *summary_out, const hl_isis_route_cell *base_cells,
                               uint32_t n_base, const uint32_t *base_of, hl_route_delta_job *job_out,
                               hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_isis_l1_to_l2_from_cells(const hl_isis_instance *l1, const hspf_isis_l1_to_l2_table *t,
                                  const hl_isis_route_cell *cells, const uint64_t *summary_words, hl_isis_ipreach *out,
                                  uint32_t cap, uint32_t *n_out);

/*
 * Backbone routers over L1 what-if jobs: the routes a level-2 router R outside an area gets from the area's L1/L2
 * routers ("borders") when a job changes costs inside the area (isis_backbone_cells.h).  Each border re-originates
 * its L2 LSP with the same IS reachability, so R's L2 SPT is its unperturbed one in every job, and only the
 * prefixes that are keys of a border's L1 -> L2 table can route differently: the affected prefixes.  Every other
 * prefix of R's table is the same in every job (hspf_isis_routes_batch over R's one row, or the host).  Out of
 * scope: R a border of the area, and jobs that also change the L2 LSDB.
 *
 *   hspf_isis_backbone_table_create  `l2` R's level-2 instance image (level_type 2, or 3 when R is an L1/L2 router
 *                             of another area); `derived` one byte per entry of l2->lvl.ipreaches (NULL: none set): a
 *                             set byte marks an entry of a border's L2 LSP that propagation or an active summary put
 *                             there; `borders` 1..8 L1 -> L2 tables (hspf_isis_l1_to_l2_table_create), which must
 *                             outlive the table.  The table holds the affected prefixes in hl_isis_rib order, each
 *                             with R's contributors in compute_routes' walk order over the LSDB where each border's
 *                             derived entries are dropped and its job's entries are appended to its zeroth fragment:
 *                             static entries read R's planes, and one slot per (border, key), at the border's vertex,
 *                             reads that border's cell of the job.  L1 -> L2 keys are plain IPv6 (MT-IPv6 entries
 *                             propagate as IPv6), so with MT-IPv6 enabled at R an IPv6 key gets no slot, as
 *                             compute_routes reads no such entry there.
 *                             HSPF_E_INVAL: wrong level or level type; 0 or more than 8 borders; R one of the
 *                             borders; two tables of the same router; a border without a valid zeroth fragment of its
 *                             non-pseudonode LSP in R's image; a derived byte outside a border's own non-pseudonode
 *                             LSP, or on an entry whose (kind, prefix) is not among that border's keys.
 *                             HSPF_E_UNSUPPORTED: a summary key of a border equal to a non-derived entry of its own
 *                             LSP (propagation would overwrite that entry).
 *   hspf_isis_backbone_table_prefixes  P, prefix[P], len[P]; any pointer may be NULL.
 *   hspf_isis_backbone_table_upload  copies the table to the ctx's device.
 *   hspf_isis_backbone_cells[16]  DEVICE planes of R's L2 batch (l2_std; l2_mt6 may be NULL unless R has an MT-IPv6
 *                             root; the wide ones with nh_words == 1): only row 0, R's unperturbed SPT, is read.
 *                             border_cells: host array of n_borders device pointers, border b's [n_jobs][K_b] cells
 *                             as hspf_isis_l1_to_l2_cells[16] wrote them for the same job order (8-byte aligned);
 *                             border_status: host array of n_borders device [n_jobs] status words (entries may be
 *                             NULL), or NULL.  cells[n_jobs][P] (device): hl_isis_route_cell as
 *                             hspf_isis_routes_batch's (lowest metric wins, equal metrics OR the next-hop atoms,
 *                             HL_CELL_CONNECTED for the root, HL_CELL_MIXED_SID for SR-relevant best contributions
 *                             from two vertices, e.g. two tying borders); winner: a static contributor's index, or
 *                             for a slot the table's contributor count + one index per (slot, border record), so a
 *                             new winning record at an equal metric is a new winner.  job_status_out (device
 *                             [n_jobs], or NULL): the OR of R's row-0 status words and the job's border status words;
 *                             a job with a non-zero status gets empty cells.  Nothing is launched for 0 jobs.
 *                             Enqueued on the ctx stream; no synchronisation.
 *   hspf_isis_backbone_delta[16]  the route-delta stage (below) over the same walk: LOST, GAINED, METRIC, NEXTHOPS
 *                             (another border takes over), OTHER.
 *   hspf_isis_backbone_from_cells  host: one job's cells -> exactly the routes of the affected prefixes that
 *                             hspf_isis_routes_from_planes gives over R's planes in the LSDB where each border's
 *                             derived entries are replaced by entries[b] (n_entries[b] of them), that border's
 *                             hspf_isis_l1_to_l2_from_cells output for the job, appended to its zeroth fragment.
 *                             planes[2]: R's planes of the standard and MT-IPv6 topologies (row 0, no overrides).
 *                             A slot's route takes its external bit and Prefix-SID from the border's entry.
 *                             HSPF_E_UNSUPPORTED for an HL_CELL_MIXED_SID cell, as hspf_isis_routes_from_cells.
 */
typedef struct hspf_isis_backbone_table hspf_isis_backbone_table;
int hspf_isis_backbone_table_create(const hl_isis_instance *l2, const uint8_t *derived, uint32_t n_borders,
                                    const hspf_isis_l1_to_l2_table *const *borders, hspf_isis_backbone_table **out);
void hspf_isis_backbone_table_free(hspf_isis_backbone_table *t);
int hspf_isis_backbone_table_prefixes(const hspf_isis_backbone_table *t, uint32_t *n_prefixes,
                                      const hl_ip_addr **prefix, const uint8_t **len);
int hspf_isis_backbone_table_upload(hspf_ctx *ctx, hspf_isis_backbone_table *t);
int hspf_isis_backbone_cells(hspf_ctx *ctx, const hspf_isis_backbone_table *t, uint32_t n_jobs,
                             const hspf_result *l2_std, const hspf_result *l2_mt6,
                             const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status,
                             uint32_t *job_status_out, hl_isis_route_cell *cells);
int hspf_isis_backbone_cells16(hspf_ctx *ctx, const hspf_isis_backbone_table *t, uint32_t n_jobs,
                               const hspf_result16 *l2_std, const hspf_result16 *l2_mt6,
                               const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status,
                               uint32_t *job_status_out, hl_isis_route_cell *cells);
int hspf_isis_backbone_delta(hspf_ctx *ctx, const hspf_isis_backbone_table *t, uint32_t n_jobs,
                             const hspf_result *l2_std, const hspf_result *l2_mt6,
                             const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status,
                             const hl_isis_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                             hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_isis_backbone_delta16(hspf_ctx *ctx, const hspf_isis_backbone_table *t, uint32_t n_jobs,
                               const hspf_result16 *l2_std, const hspf_result16 *l2_mt6,
                               const hl_isis_route_cell *const *border_cells, const uint32_t *const *border_status,
                               const hl_isis_route_cell *base_cells, uint32_t n_base, const uint32_t *base_of,
                               hl_route_delta_job *job_out, hl_route_delta *records, uint64_t cap, uint64_t *n_records);
int hspf_isis_backbone_from_cells(const hl_isis_instance *l2, const hspf_isis_backbone_table *t,
                                  const hl_isis_route_cell *cells, const hspf_isis_job_planes *planes,
                                  const hl_isis_ipreach *const *entries, const uint32_t *n_entries, hl_isis_rib *out);

/*
 * Route-delta stage on the device: which prefixes each job of a what-if batch loses, gains, or reaches at another
 * metric or over another next-hop set, against a base route table — without storing the n_jobs x P cell matrix.
 * Per (job, prefix) it runs the same walk as hspf_*_routes_batch[16] and compares the cell with the job's base cell
 * word for word (for a fixed root, atom a is always the same first hop, whatever the job's overrides).  Enqueued on
 * the ctx stream behind the SPT batches; no synchronisation.  One call covers at most 2^36 cells: every route-delta
 * entry point (hspf_*_delta[16], here and above) returns HSPF_E_INVAL and enqueues nothing when n_jobs x P > 2^36,
 * P being the table's prefixes (its keys for hspf_isis_l1_to_l2_delta); a caller splits a larger sweep into several
 * calls.
 *
 *   hspf_ospfv2_routes_delta[16]  OSPFv2 and OSPFv3 tables (as hspf_ospfv2_routes_batch[16]).
 *   hspf_isis_routes_delta[16]    IS-IS tables (as hspf_isis_routes_batch[16]).
 *   hspf_ospfv2_rib_delta[16]     OSPFv2 and OSPFv3 routing tables (as hspf_ospfv2_rib_cells[16]: the wide call needs
 *                                 nh_words == 1; roots: device u32[n_jobs], required when n_jobs > 0).  A job and
 *                                 its base row must share a root: atoms compare word for word only then.  The base
 *                                 row is normally hspf_ospfv2_rib_cells over the root's unperturbed job.
 *   base_cells  DEVICE [n_base][P] cells, 8-byte aligned: typically written by hspf_*_routes_batch[16] for the
 *               unperturbed job of each root.  n_base == 0 is HSPF_E_INVAL.
 *   base_of     DEVICE [n_jobs] base row of each job, or NULL: every job uses row 0.
 *   job_out     DEVICE [n_jobs] hl_route_delta_job (required).  status: the job's status word (IS-IS: both
 *               topologies' OR-ed; routing tables: what job_status_out of hspf_ospfv2_rib_cells holds), or
 *               HSPF_JS_INVALID when base_of[j] >= n_base.  A job with a non-zero status is not compared: counts 0,
 *               no records.
 *   records     DEVICE hl_route_delta[cap], ordered by (job, prefix), identical from run to run.  Only the first
 *               min(total, cap) are written.  records NULL or cap 0: the summaries only.
 *   n_records   DEVICE uint64_t (required): the total number of changed (job, prefix), whatever cap is.
 *
 * Kinds (include/holo_lsdb.h, HL_DELTA_*), with B the base cell and J the job cell: LOST (B present, J not),
 * GAINED (J present, B not); both present: METRIC, NEXTHOPS (nh_mask), OTHER (winner or flags; OSPF: also
 * lasthop_mask) in any combination; neither present: no change.  Routing-table cells (hl_ospf_rib_cell): METRIC is
 * the 26-bit cell metric (for a type-2 external, the forwarding metric to the ASBR, not the type-2 metric); OTHER is
 * a changed winner, path type, HL_CELL_* flags or aux (intra-area last-hop atoms, or the type-2 metric, which the
 * winner fixes).  A new path type always comes with a new winner, so it is OTHER; a caller who needs the path type
 * decodes the job (hspf_ospfv2_rib_from_cells).  What is not promised: an unchanged cell does not
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
int hspf_ospfv2_rib_delta(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result *planes,
                          const uint32_t *roots, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                          const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records,
                          uint64_t cap, uint64_t *n_records);
int hspf_ospfv2_rib_delta16(hspf_ctx *ctx, const hspf_ospfv2_ribtable *rt, uint32_t n_jobs, const hspf_result16 *planes,
                            const uint32_t *roots, const hl_ospf_rib_cell *base_cells, uint32_t n_base,
                            const uint32_t *base_of, hl_route_delta_job *job_out, hl_route_delta *records,
                            uint64_t cap, uint64_t *n_records);

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
