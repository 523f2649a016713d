// Routing table of an OSPF backbone router R for a batch of what-if jobs inside other areas, one cell per (job,
// affected prefix) (include/holo_spf_lsdb.h, hspf_ospfv2_backbone_table_create / hspf_ospfv3_backbone_table_create).
//
// A job changes costs only in the non-backbone areas of the area border routers given as "borders".  R is an
// internal router of area 0, so its area-0 SPT is its unperturbed one in every job, and only the type-3 /
// Inter-Area-Prefix LSAs the borders originate into area 0 change.  Only a prefix some border can advertise (one with
// an intra-area record in one of the border's non-backbone areas) can route differently at R.  Per such prefix the
// walk is ospf_rib_cell_eval (ospf_rib_cells.h) over R's row 0, with each border's LSA for the prefix replaced by a
// slot at that border's place in LsaKey order:
//   * a static type-3 record reads R's planes as before (dist[abr] + metric);
//   * a slot reads the border's routing-table cell of the job (ospf_abr_rib_cells.h) and stands for the LSA
//     compute_net_summaries (holo-ospf area.rs:561-659) originates into the backbone: the cell is present and
//     intra-area, its winner is not one of area 0's intra-area records (route.area_id != 0), none of its atoms is an
//     area-0 atom (nexthops_area_check, area.rs:742) and its metric is below LSInfinity.  Then it offers
//     dist[border] + the cell's metric.
// The lowest metric wins and equal metrics OR their atoms, the first record staying the winner.  A slot's winner
// is n_recs + its slot index (OSPFv2), so the decode can tell it from a static record.  An OSPFv3 slot also carries
// the prefix options the border copies from its route into the LSA (lsa_orig_inter_area_network, ospfv3/lsdb.rs:
// 341-386): those of the border cell's winning intra-area record.  Its winner is n_recs + (slot << 8 | options), so
// that a job whose border route changes record at an equal metric, to one with other options, changes R's winner
// (the route-delta stage reports OTHER), and the decode reads the options from the winner alone.
//
// The same walk serves the opposite direction (kNonBackbone, hspf_ospfv2_nonbackbone_table_create): R is an internal
// router of a non-backbone area A, a job changes costs in area 0 only, and the borders are A's ABRs attached to area
// 0.  A slot then stands for the LSA the border originates into A: its cell may also be inter-area, its winner must
// not be one of A's intra-area records and none of its atoms an A atom.
#pragma once
#include <cstdint>
#include <utility>
#include <vector>

#include "ospf_abr_rib_cells.h"

namespace hspf {

constexpr uint32_t kOspfBackboneMaxBorders = 8;
constexpr uint32_t kOspfBackboneStatic = 0xFFFFFFFFu;   // RibRec::z of a static type-3 record

// Whether a table's cell winners fit their u32 below kNoRecord: a slot's winner is n_recs + its slot index (OSPFv3:
// n_recs + (slot index << 8 | prefix options)).  A table that does not is refused (HSPF_E_UNSUPPORTED).  Host only.
inline bool backbone_winners_fit(uint64_t n_recs, uint64_t n_slots, bool v3) {
    return n_recs + (v3 ? n_slots << 8 : n_slots) < 0xFFFFFFFFull;
}

// Type-3 records of the backbone table, beside R's one-area records (ospf_rib_cells.h):
//   static: x ABR vertex, y LSA metric, z kOspfBackboneStatic
//   slot:   x the border's vertex, y the prefix's index in the border's table, z the border, w the slot index

// What the walk reads of a table.  Per border b, border[4 b ..] (OSPFv2) or border[8 b ..] (OSPFv3): its area-0
// intra-area records [lo, hi) and its area-0 atom bits (low word, high word); OSPFv3 adds the byte offset, from
// `border`, of the border's options bytes, one per intra-area record of its table (the winner of an intra-area cell
// indexes them), then three zero words (an OSPFv3 third-area table: C's record count, then two zero words, and C's
// options bytes cover every record index below that count).
struct OspfBackboneView {
    const uint32_t *oi;           // [PR + 1] R's intra-area ranges (R's one-area table)
    const uint32_t *q;            // [P] the prefix's index in R's one-area table, kNoRecord if none
    const uint32_t *o3;           // [P + 1] type-3 ranges (statics and slots)
    const uint32_t *o5;           // [P + 1] type-5 ranges
    const uint32_t *border;       // [4 n_borders]
    const RibRec *recs;
    uint32_t P, n_recs, root;
};

// One job's row of every border's cells.
struct OspfBorderRows {
    const hl_ospf_rib_cell *row[kOspfBackboneMaxBorders];
};

// Type-4 slots (OSPFv2, hspf_ospfv2_backbone_asbr_table_create).  A border originates a type-4 LSA into area 0 for an
// ASBR A (compute_rtr_summaries, ospf_rib_host.cc: hspf_ospfv2_net_summaries) when A is a router of one of its
// non-backbone areas with the E flag and the border reaches A in that area below LSInfinity; its metric is that
// distance, and an id in two such areas keeps the later area's entry.  In R's type-4 range for A (walked from the end,
// as rib_full's step 2 lets the last usable LSA replace the entry) each border has one slot per such area, in area
// order, at the border's place in LsaKey order:
//   static: x ABR vertex, y LSA metric, z 0, w 0 (as in ospf_rib_cells.h)
//   slot:   x the border's vertex, y A's vertex in the slot's area, z the border, w kOspfBackboneAsbrSlot | plane set
// A plane set is one (border, non-backbone area) pair; a call reads at most kOspfBackboneMaxAsbrSets of them.
constexpr uint32_t kOspfBackboneMaxAsbrSets = 8;
constexpr uint32_t kOspfBackboneAsbrSlot = 0x80000000u;

// The plane sets a table's type-4 slots read: set k is area `area[k]` of a border whose rows are rows[k][job][stride[k]]
// (< n_rows[k]), each row V[k] vertices of dist[k] and a status word (status[k] may be NULL).
template <class D>
struct OspfAsbrSets {
    const D *dist[kOspfBackboneMaxAsbrSets];
    const uint32_t *status[kOspfBackboneMaxAsbrSets];
    const uint32_t *rows[kOspfBackboneMaxAsbrSets];
    uint32_t V[kOspfBackboneMaxAsbrSets], n_rows[kOspfBackboneMaxAsbrSets];
    uint32_t stride[kOspfBackboneMaxAsbrSets], area[kOspfBackboneMaxAsbrSets];
    uint32_t n;
    HSPF_HD uint32_t row(uint32_t k, uint32_t j) const { return rows[k][(size_t)j * stride[k] + area[k]]; }
};

// The OR of the job's rows' status words over the sets, HSPF_JS_INVALID for a row out of range (read before any plane).
template <class D>
HSPF_HD uint32_t asbr_job_status(const OspfAsbrSets<D> &s, uint32_t j) {
    uint32_t st = 0;
    for (uint32_t k = 0; k < s.n; ++k) {
        const uint32_t r = s.row(k, j);
        if (r >= s.n_rows[k]) st |= HSPF_JS_INVALID;
        else if (s.status[k]) st |= s.status[k][r];
    }
    return st;
}

// One job of the sets: whether the border of set k originates a type-4 LSA for the ASBR at vertex v of its area, and
// at what metric.  The intra-area entry of a non-backbone area only has that area's next hops, so the rule that no
// next hop may be on an area-0 interface (nexthops_area_check) always holds here.
template <class Planes, class D>
struct OspfAsbrJob {
    const OspfAsbrSets<D> &s;
    uint32_t j;
    HSPF_HD bool originates(uint32_t k, uint32_t v, uint32_t &metric) const {
        const Planes pl{s.dist[k] + (size_t)s.row(k, j) * s.V[k], nullptr, nullptr};
        if (!pl.reached(v)) return false;
        metric = pl.d(v);
        return metric < HL_LSA_INFINITY;
    }
};

// R's planes of a job over a table with type-4 slots, with the job's plane sets beside them.  (The accessor rides
// with the planes, which stay in registers, and not with the border rows, which the walk indexes at run time: a
// reference to the kernel parameter stored there would copy the whole parameter to local memory.)
template <class Planes, class D>
struct OspfAsbrPlanes : Planes {
    OspfAsbrJob<Planes, D> asbr;
};

// What border b advertises into the table's target area for the prefix of its cell c: false when nothing, else its
// metric and, for OSPFv3 (kV3), the prefix options of the cell's winner.  Into area 0 only an intra-area route is
// advertised; into a non-backbone area (kNonBackbone, hspf_ospfv2_nonbackbone_table_create) an inter-area one too
// (compute_net_summaries).  The border words name the target area's intra-area records and atoms.
// kSlotWinners (OSPFv3 third-area tables, hspf_ospfv3_third_area_table_create): the border's cells are those of an
// OSPFv3 abr_backbone table, whose inter-area winners from its own slots are n_recs_C + (slot << 8 | options).  The
// border's sixth word is n_recs_C: a winner at or above it carries its options in the low byte of winner - n_recs_C,
// and a record winner (an intra-area walk record, a static Inter-Area-Prefix record) reads them from the options
// bytes.
template <bool kV3, bool kNonBackbone = false, bool kSlotWinners = false>
HSPF_HD bool border_summary(const hl_ospf_rib_cell *c, const uint32_t *border, uint32_t b, uint32_t &metric,
                            uint32_t &options) {
    constexpr uint32_t kStride = kV3 ? 2 : 1;                          // 16-byte groups per border
#if defined(__CUDA_ARCH__)
    const unsigned long long *w = reinterpret_cast<const unsigned long long *>(c);
    const uint64_t wm = __ldg(w + 2), nh = __ldg(w);
    const uint4 bb = __ldg(reinterpret_cast<const uint4 *>(border) + kStride * b);
#else
    const uint64_t wm = (uint64_t)c->winner | ((uint64_t)c->mpf << 32), nh = c->nh_mask;
    const uint32_t *bw = border + 4 * kStride * b;
    const struct { uint32_t x, y, z, w; } bb = {bw[0], bw[1], bw[2], bw[3]};
#endif
    const uint32_t winner = (uint32_t)wm, mpf = (uint32_t)(wm >> 32);
    const uint64_t atoms0 = (uint64_t)bb.z | ((uint64_t)bb.w << 32);
    metric = mpf & HL_RIB_CELL_METRIC_MAX;
    const uint32_t path = (mpf >> 26) & 0x3u;
    const bool adv = ((mpf >> 28) & HL_CELL_PRESENT) &&
                     (path == HL_PATH_INTRA_AREA || (kNonBackbone && path == HL_PATH_INTER_AREA)) &&
                     (winner < bb.x || winner >= bb.y) && !(nh & atoms0) && metric < HL_LSA_INFINITY;
    if constexpr (kV3) {
        options = 0;
        if constexpr (kSlotWinners) {
            if (adv) {
#if defined(__CUDA_ARCH__)
                const uint2 ow = __ldg(reinterpret_cast<const uint2 *>(border + 8 * b + 4));
                options = winner >= ow.y ? ((winner - ow.y) & 0xFFu)
                                         : __ldg(reinterpret_cast<const uint8_t *>(border) + ow.x + winner);
#else
                const uint32_t n = border[8 * b + 5];
                options = winner >= n ? ((winner - n) & 0xFFu)
                                      : reinterpret_cast<const uint8_t *>(border)[border[8 * b + 4] + winner];
#endif
            }
        } else if (adv) {
#if defined(__CUDA_ARCH__)
            options = __ldg(reinterpret_cast<const uint8_t *>(border) + __ldg(border + 8 * b + 4) + winner);
#else
            options = reinterpret_cast<const uint8_t *>(border)[border[8 * b + 4] + winner];
#endif
        }
    }
    return adv;
}

// kV3: the table is an OSPFv3 one (hspf_ospfv3_backbone_table_create), whose slot winners carry prefix options.
// kAsbr: the table's type-4 ranges hold slots, read through pl.asbr (pl an OspfAsbrPlanes of the job).
// kNonBackbone: the table's target area is not area 0 (border_summary).
// kSlotWinners: the borders' cells may hold OSPFv3 slot winners (border_summary; an OSPFv3 third-area table).
template <bool kV3 = false, bool kAsbr = false, bool kNonBackbone = false, bool kSlotWinners = false, class Planes>
HSPF_HD CellWords ospf_backbone_cell_eval(const Planes &pl, const OspfBackboneView &t, uint32_t p,
                                          const OspfBorderRows &rows) {
    const RouteContrib *contribs = reinterpret_cast<const RouteContrib *>(t.recs);
    const uint32_t q = t.q[p];
    if (q != kNoRecord) {                                               // 1. intra-area
        const hl_route_cell c = route_cell_eval(pl, contribs, t.oi[q], t.oi[q + 1]);
        if (c.flags & HL_CELL_PRESENT)
            return {c.nh_mask, c.lasthop_mask, (uint64_t)c.winner | ((uint64_t)rib_mpf(c.metric, HL_PATH_INTRA_AREA, c.flags) << 32)};
    }
    uint64_t mask = 0;
    uint32_t win = kNoRecord, metric = 0;
    for (uint32_t i = t.o3[p]; i < t.o3[p + 1]; ++i) {                  // 2. inter-area, slots in LsaKey order
        const RibRec r = load_rib_rec(t.recs + i);
        if (!pl.reached(r.x)) continue;
        uint32_t y = r.y, w = i, options = 0;
        if (r.z != kOspfBackboneStatic) {
            if (!border_summary<kV3, kNonBackbone, kSlotWinners>(rows.row[r.z] + r.y, t.border, r.z, y, options))
                continue;
            w = kV3 ? t.n_recs + (r.w << 8 | options) : t.n_recs + r.w;
        }
        const uint32_t m = pl.d(r.x) + y;
        if (win == kNoRecord || m < metric) { win = w; metric = m; mask = pl.n(r.x); }
        else if (m == metric) mask |= pl.n(r.x);
    }
    if (win != kNoRecord)
        return {mask, 0, (uint64_t)win | ((uint64_t)rib_mpf(metric, HL_PATH_INTER_AREA, HL_CELL_PRESENT) << 32)};
    uint32_t path = 0, type2 = 0;
    for (uint32_t i = t.o5[p]; i < t.o5[p + 1]; ++i) {                  // 3. AS-external, as ospf_rib_cell_eval
        const RibRec r = load_rib_rec(t.recs + i);
        const RibRec s = load_rib_rec(t.recs + r.x);
        if (s.x == t.root) continue;
        uint32_t em = 0;
        uint64_t en = 0;
        bool have = false;
        for (uint32_t k = s.w; k > s.z; --k) {
            const RibRec f = load_rib_rec(t.recs + k - 1);
            if (f.x == t.root || !pl.reached(f.x)) continue;
            if constexpr (kAsbr) {
                uint32_t fm = f.y;                                      // a border that does not originate: go on
                if ((f.w & kOspfBackboneAsbrSlot) && !pl.asbr.originates(f.w & ~kOspfBackboneAsbrSlot, f.y, fm)) continue;
                em = pl.d(f.x) + fm;
            } else {
                em = pl.d(f.x) + f.y;
            }
            en = pl.n(f.x); have = true;
            break;
        }
        if (!have) {
            if (!s.y || !pl.reached(s.x)) continue;
            em = pl.d(s.x); en = pl.n(s.x);
        }
        const uint32_t cp = r.z ? HL_PATH_TYPE2_EXTERNAL : HL_PATH_TYPE1_EXTERNAL;
        const uint32_t cm = r.z ? em : em + r.y, c2 = r.z ? r.y : 0;
        int cmp = -1;
        if (win != kNoRecord) {
            if (cp != path) cmp = cp < path ? -1 : 1;
            else if (cp == HL_PATH_TYPE2_EXTERNAL && c2 != type2) cmp = c2 < type2 ? -1 : 1;
            else cmp = cm < metric ? -1 : (cm == metric ? 0 : 1);
        }
        if (cmp < 0) { win = i; path = cp; metric = cm; type2 = c2; mask = en; }
        else if (cmp == 0) mask |= en;
    }
    if (win == kNoRecord) return {0, 0, (uint64_t)kNoRecord};
    return {mask, type2, (uint64_t)win | ((uint64_t)rib_mpf(metric, path, HL_CELL_PRESENT) << 32)};
}

// An area border router R over jobs inside an area it is not attached to (hspf_ospfv2_abr_backbone_table_create):
// abr_rib_cell_eval with kSlots over R's row 0 of every area.  Area 0's type-3 ranges hold static records (z
// kOspfBackboneStatic) and slots as the backbone table's, its type-4 ranges static records and type-4 slots as the
// asbr table's.  A slot's winner is n_recs + its slot index; kV3 (hspf_ospfv3_abr_backbone_table_create): n_recs +
// (slot index << 8 | prefix options), as ospf_backbone_cell_eval<kV3> gives it.
template <bool kV3 = false>
struct AbrBorderSlots {
    static constexpr uint32_t kAsbrSlot = kOspfBackboneAsbrSlot;
    OspfBorderRows rows;
    const uint32_t *border;       // [4 n_borders] (OSPFv3: [8 n_borders] and the options bytes) as OspfBackboneView::border
    uint32_t n_recs;
    // what type-3 record r offers: a static one its own metric, a slot its border's advertisement (false: none)
    HSPF_HD bool offer(const RibRec &r, uint32_t &metric, uint32_t &winner) const {
        if (r.z == kOspfBackboneStatic) return true;
        uint32_t options;
        if (!border_summary<kV3>(rows.row[r.z] + r.y, border, r.z, metric, options)) return false;
        winner = kV3 ? n_recs + (r.w << 8 | options) : n_recs + r.w;
        return true;
    }
};

// R's planes of area i at row 0, and the job's type-4 plane sets (kept with the planes, as OspfAsbrPlanes).
template <class Planes, class D, class N>
struct AbrRow0Planes {
    const AbrPlaneSet<D, N> &s;
    OspfAsbrJob<Planes, D> asbr;
    HSPF_HD Planes operator()(uint32_t i) const { return Planes{s.dist[i], s.hops[i], s.nh[i]}; }
};

// The OR of R's row-0 status words over its areas.
template <class D, class N>
HSPF_HD uint32_t abr_row0_status(const AbrPlaneSet<D, N> &s, uint32_t n_areas) {
    uint32_t st = 0;
    for (uint32_t i = 0; i < n_areas; ++i)
        if (s.status[i]) st |= s.status[i][0];
    return st;
}

// ---- a non-backbone router over jobs inside another non-backbone area (hspf_ospfv2_third_area_table_create) --------
// R is an internal router of area 2, the jobs perturb area 1, and the borders are area 2's ABRs attached to area 0
// (C), each an hspf_ospfv2_abr_backbone_table over area 1's ABRs (B).  A type-3 slot reads C's cell of the job as a
// kNonBackbone slot does.  When area 1 holds an ASBR A, C's area-0 entry for A is inter-area, through the B's type-4
// LSAs, and moves with the job; so does the metric of the type-4 LSA C originates for A into area 2.  R's type-4 range
// for A then holds one chain slot per C, at C's place in LsaKey order:
//   chain slot: x C's vertex, y the group's index among C's groups with type-4 slots, z C, w kOspfBackboneAsbrSlot | C
// and the walk reads C's entry of the job (abr_asbr_entry below, stored by hspf_ospfv2_abr_backbone_asbr_entries).
// OSPFv3 (hspf_ospfv3_third_area_table_create): C copies its route's prefix options into the Inter-Area-Prefix LSA it
// originates, and C's inter-area routes come from the B's slots, whose winners carry the options (n_recs_C + (slot << 8
// | options)); the walk reads them with kSlotWinners (border_summary).  C's Inter-Area-Router ranges hold the same
// records as OSPFv2's type-4 ranges, so abr_asbr_entry serves both versions.
constexpr uint32_t kOspfNoEntry = 0xFFFFFFFFu;        // an entry C does not originate a type-4 LSA for

// C's area-0 entry of an ASBR, as rib_full step 2 leaves it and compute_rtr_summaries re-originates it into a normal
// area: the last type-4 record of the entry's range (`e`, an ASBR entry record of C's area 0) whose ABR C reaches and,
// for a type-4 slot, whose border originates (asbr), else the ASBR's own vertex with the E flag; its metric, or
// kOspfNoEntry when there is none or it is not below LSInfinity.  The same loop as abr_rib_cell_eval's step 4 for one
// area, kept apart so that the kernels over that walk keep their code.
template <class Planes, class D>
HSPF_HD uint32_t abr_asbr_entry(const Planes &pl, const OspfAsbrJob<Planes, D> &asbr, const RibRec *recs, uint32_t e) {
    const RibRec s = load_rib_rec(recs + e);
    uint32_t m = kOspfNoEntry;
    bool found = false;
    for (uint32_t k = s.w; k > s.z && !found; --k) {
        const RibRec f = load_rib_rec(recs + k - 1);
        if (!pl.reached(f.x)) continue;
        uint32_t fm = f.y;
        if ((f.w & kOspfBackboneAsbrSlot) && !asbr.originates(f.w & ~kOspfBackboneAsbrSlot, f.y, fm)) continue;
        m = pl.d(f.x) + fm; found = true;
    }
    if (!found && s.y && pl.reached(s.x)) m = pl.d(s.x);
    return m < HL_LSA_INFINITY ? m : kOspfNoEntry;
}

// Each C's entries of the jobs, u32 [n_jobs][G[b]] (kOspfNoEntry: no type-4 LSA), and their status words (may be NULL).
struct OspfChainSet {
    const uint32_t *entries[kOspfBackboneMaxBorders];
    const uint32_t *status[kOspfBackboneMaxBorders];
    uint32_t G[kOspfBackboneMaxBorders];
};

// One job of the set, as OspfAsbrJob: whether C (b) originates a type-4 LSA for its group g, and at what metric.
struct OspfChainJob {
    const OspfChainSet &s;
    uint32_t j;
    HSPF_HD bool originates(uint32_t b, uint32_t g, uint32_t &metric) const {
#if defined(__CUDA_ARCH__)
        metric = __ldg(s.entries[b] + (size_t)j * s.G[b] + g);
#else
        metric = s.entries[b][(size_t)j * s.G[b] + g];
#endif
        return metric != kOspfNoEntry;
    }
};

// R's planes of a job over a table with chain slots, with the job's entries beside them (as OspfAsbrPlanes).
template <class Planes>
struct OspfThirdAreaPlanes : Planes {
    OspfChainJob asbr;
};

}  // namespace hspf

// Host + device image of an area border router's affected prefixes over jobs inside another area
// (include/holo_spf_lsdb.h, hspf_ospfv{2,3}_abr_backbone_table_create; ospf_ribtable.h, build_abr_backbone_table).
struct hspf_ospfv2_abr_backbone_table {
    // R's table over the affected prefixes.  Its records: every area's intra-area records as R's whole table has them
    // (the decode's), the type-3 ranges (area 0's with slots), the type-5 ranges, the ASBR entries and type-4 ranges,
    // then from walk_intra the intra-area records of the affected prefixes again, which `off` names for the walk.
    // abr->v3 marks an OSPFv3 table: its options6 holds a placeholder for each slot, whose options come from its winner.
    hspf_ospfv2_abr_ribtable *abr = nullptr;
    uint32_t area0 = 0, n_borders = 0, walk_intra = 0;
    const hspf_ospfv2_abr_ribtable *borders[hspf::kOspfBackboneMaxBorders] = {};
    std::vector<uint32_t> intra_src;             // per walk intra-area record (index - walk_intra): the decode's record
    std::vector<uint32_t> slot_rec;              // [n_slots] the record of each slot
    uint32_t n_asbr_slots = 0;
    std::vector<std::pair<uint32_t, uint32_t>> asbr_set;   // the type-4 slots' plane sets (border, area index)
    std::vector<uint32_t> words;                 // abr->off, padded to 16 bytes, then border [4 n_borders] (OSPFv3:
                                                 // [8 n_borders], then each border's options bytes)
    hspf::DeviceRouteTable dev;                  // words, then records
    // the ASBR entry groups whose area-0 type-4 range holds type-4 slots, ascending: the entries
    // hspf_ospfv2_abr_backbone_asbr_entries computes, and the chain slots of a third-area table
    std::vector<uint32_t> asbr_group, asbr_group_id;   // ... and each one's ASBR id
    hspf::DeviceRouteTable entry_dev;            // per such group its area-0 entry record (uploaded when there is one)

    uint32_t P() const { return (uint32_t)abr->prefix.size(); }
    uint32_t n_recs() const { return (uint32_t)abr->recs.size(); }
    size_t border_at() const { return (abr->off.size() + 3) & ~(size_t)3; }
    hspf::AbrRibView view(const uint32_t *w, const hspf::RibRec *rc) const {
        return abr->view(w, rc, reinterpret_cast<const uint32_t *>(rc + abr->recs.size()));
    }
};

// Host + device image of a backbone router's affected prefixes (include/holo_spf_lsdb.h).
struct hspf_ospfv2_backbone_table {
    hspf_ospfv2_ribtable *r = nullptr;           // R's one-area table over its area without the borders' type-3 LSAs
    uint32_t router_id = 0, root = 0, n_vertices = 0, n_borders = 0, max_paths = 0;
    // the target area: R's area, into which the borders' LSAs are re-originated per job (0 but for
    // hspf_ospfv2_nonbackbone_table_create, whose tables the walk reads with kNonBackbone)
    uint32_t area_id = 0;
    std::vector<uint32_t> prefix, plen;          // [P] prefix order
    // oi [PR + 1], q [P], o3 [P + 1], o5 [P + 1], padding, border [4 n_borders] (OSPFv3: [8 n_borders], then each
    // border's options bytes, each border's padded to a word)
    std::vector<uint32_t> words;
    std::vector<hspf::RibRec> recs;              // R's records, then the type-3 and type-5 records of the view
    std::vector<uint32_t> slot_rec;              // [n_slots] the record of each slot
    std::vector<uint32_t> ext_tag;               // per type-5 record of the view (index - ext_base)
    uint32_t ext_base = 0;
    const hspf_ospfv2_abr_ribtable *borders[hspf::kOspfBackboneMaxBorders] = {};
    // hspf_ospfv2_backbone_asbr_table_create: the type-4 slot count and the plane sets they read, (border, area index
    // in the border's table); a table with type-4 slots is read only by the asbr calls
    uint32_t n_asbr_slots = 0;
    std::vector<std::pair<uint32_t, uint32_t>> asbr_set;
    // made by a create that re-originates the borders' type-4 / Inter-Area-Router LSAs per job (the asbr and
    // nonbackbone creates): the asbr calls take an OSPFv3 table of area 0 only with this mark
    bool asbr = false;
    // OSPFv3 tables (hspf_ospfv3_backbone_table_create): `prefix` is zero-filled (the prefixes are prefix6), and
    // options6 holds the prefix options of each type-3 / type-5 record of the view (index - o3[0]); a slot's entry is
    // a placeholder, its options come from its winner
    bool v3 = false;
    std::vector<hl_ip_addr> prefix6;
    std::vector<uint8_t> options6;
    // hspf_ospfv2_third_area_table_create: the borders are C tables (borders[b] is third[b]->abr), and the type-4
    // slots are chain slots (n_asbr_slots of them, no plane set), read by the third-area calls only; an OSPFv3 one
    // (hspf_ospfv3_third_area_table_create, v3 set) is read by the third-area calls only, with or without them
    bool third_area = false;
    const hspf_ospfv2_abr_backbone_table *third[hspf::kOspfBackboneMaxBorders] = {};
    hspf::DeviceRouteTable dev;                  // hspf_ospfv2_backbone_table_upload: words, then records

    uint32_t P() const { return (uint32_t)prefix.size(); }
    // the border words start on a 16-byte boundary (one 16-byte load per border)
    size_t border_at() const { return ((r->prefix.size() + 1 + 3 * (size_t)P() + 2) + 3) & ~(size_t)3; }
    hspf::OspfBackboneView view(const uint32_t *w, const hspf::RibRec *rc) const {
        const uint32_t PR = (uint32_t)r->prefix.size(), n = P();
        hspf::OspfBackboneView v;
        v.oi = w;
        v.q = w + PR + 1;
        v.o3 = v.q + n;
        v.o5 = v.o3 + n + 1;
        v.border = w + border_at();
        v.recs = rc;
        v.P = n;
        v.n_recs = (uint32_t)recs.size();
        v.root = root;
        return v;
    }
    hspf::OspfBackboneView host_view() const { return view(words.data(), recs.data()); }
};
