// The interface between the engine (lwse_engine.cu) and the kernel files (lwse_*_kernels.cu): every
// launcher, scratch-size function and argument struct one file defines and another calls.  Host
// declarations only.  Each struct is defined here and nowhere else, so that the engine and the
// kernel that reads it cannot disagree on its layout.
//
// A launcher enqueues its kernels on the stream it is given and returns the number of kernels it
// launched (>= 0), or the CUDA error it met, negated (-(int)err).  A launcher that calls another
// passes the callee's negative result through unchanged.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/lwse.h"

namespace lwse {

// A launcher returns the kernels it enqueued (>= 0), or the CUDA error it met, negated.
inline int launch_result(int kernels) {
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? kernels : -(int)e;
}

// ---- lwse_lws_kernels.cu ----
int pick_tile(uint64_t items, uint64_t owners);  // lanes per object of the LWS pass (and of the forecast)

struct SweepChangeLists {  // device (or mapped host) pointers; all null = off
  uint32_t* lws_rows = nullptr;
  lwse_lws_out* lws_out = nullptr;
  uint32_t lws_capacity = 0;
  uint32_t* group_rows = nullptr;
  lwse_group_out* group_out = nullptr;
  uint32_t group_capacity = 0;
  uint32_t* counts = nullptr;  // device: [0] lws, [1] groups; zeroed by the caller (a tick's publish kernel resets them)
};
int launch_lws_sweep(const lwse_lws_tables* t, const lwse_node_rec* d_nodes, uint32_t n_nodes,
                     void* scratch, int sm_count, cudaStream_t s, const SweepChangeLists* cl,
                     uint32_t* d_event_count = nullptr, int first_mode = 1);
size_t lws_sweep_scratch_bytes(uint64_t n_pods, uint32_t n_groups);
// The sweep scratch's flag column: one byte per group row, the low five bits of its group_out.flags, which
// the group pass writes and the LWS pass reads.
uint8_t* lws_sweep_flag_column(void* scratch, uint64_t n_pods);

struct PublishListHost {
  const uint32_t* src_rows;
  const void* src_outs;
  uint32_t* dst_rows;
  void* dst_outs;
  uint32_t* count;   // null = skip this slot
  uint32_t capacity;
  uint32_t out_bytes;
};
int launch_publish(const PublishListHost* lists, const uint32_t* d_extra, uint32_t* h_words, uint32_t seq_slot,
                   uint32_t seq, uint32_t* d_ticket, uint32_t expected_rows, cudaStream_t s,
                   uint32_t* d_clear, uint32_t n_clear, bool pdl);

struct ScatterSegHost {
  void* table;
  uint64_t table_rows;
  const uint32_t* rows;
  const void* values;
  uint32_t n;
  uint32_t row_bytes;
  bool is_ident;
};
int launch_scatter(const ScatterSegHost* segs, int n_segs, uint32_t* d_occupancy, uint32_t n_nodes, cudaStream_t s,
                   bool pdl);
// Bytes of one scatter descriptor block of a graph tick (write_scatter_desc / launch_scatter_desc); the
// kernel file asserts that its argument block fits.
constexpr size_t kScatterDescBytes = 512;
bool write_scatter_desc(void* h_desc, const ScatterSegHost* segs, int n_segs, uint32_t* d_occupancy, uint32_t n_nodes);
int launch_scatter_desc(const void* d_desc, int sm_count, cudaStream_t s, bool pdl);
int launch_ident_prefetch(const uint8_t* d_state, uint64_t n_pods, const lwse_pod_ident* mapped_host_ident,
                          lwse_pod_ident* d_ident, int sm_count, cudaStream_t s);
int launch_occupancy(const lwse_pod_ident* d_ident, uint64_t n_pods, uint32_t* d_occupancy, uint32_t n_nodes, int sm_count,
                     cudaStream_t s);

// ---- lwse_place_kernels.cu ----
int launch_place(const lwse_node_rec* d_nodes, const uint32_t* d_dom_first, const uint32_t* d_node_order,
                 const uint32_t* d_node_pos, uint32_t n_nodes, uint32_t n_domains,
                 const lwse_place_req* d_reqs, uint32_t n_reqs, const uint32_t* d_occupancy,
                 uint32_t n_namespaces, lwse_place_out* d_out, void* d_scratch, size_t scratch_bytes,
                 uint32_t* h_rounds, int sm_count, cudaStream_t s, uint32_t call_index,
                 bool fresh, uint32_t n_parts, uint32_t reqs_per_part, uint64_t part_stride_bytes,
                 uint32_t* h_unpinned, const uint32_t** d_counters_out, const uint32_t** d_unpinned_out,
                 bool after_push);
size_t place_scratch_bytes(uint32_t n_nodes, uint32_t n_domains, uint32_t n_reqs, uint32_t n_namespaces);
int launch_place_diff(const lwse_place_out* d_cur, lwse_place_out* d_prev, uint32_t n, uint32_t* d_rows,
                      lwse_place_out* d_outs, uint32_t capacity, uint32_t* d_count, cudaStream_t s);

// ---- lwse_place_ns_kernels.cu ----
struct PlaceNsChanges {  // a tick's change list (device memory); prev == null: off
  lwse_place_out* prev;
  uint32_t* rows;
  lwse_place_out* outs;
  uint32_t* count;
  uint32_t capacity;
  int tick_slot;  // 0 / 1: the round's counters live in the tick slot's own block, which the tick's publish
                  // kernel clears after reading (two ticks may be in flight); -1: the two alternating blocks
  void* mid_event;  // cudaEvent_t or null: recorded between the condense and the namespace kernel (a tick graph
                    // holds the sweep back until then, so that both branches reach the SMs together)
};

struct PlaceNsExchange {  // multi-rank: d_occupancy is the base of the exchange buffers (see PlaceNsArgs::xch_step)
  const unsigned long long* step_ctr;
  uint64_t half_bytes;
  bool lagged;
};

// index: kNsIndexNone = the request table is grouped by namespace; otherwise the indexed form, with the
// index kept in the scratch (kNsIndexReuse: as the last build left it — the caller knows the namespace
// column has not changed since; kNsIndexBuild: built first).
enum PlaceNsIndex : uint32_t { kNsIndexNone = 0, kNsIndexReuse = 1, kNsIndexBuild = 2 };

bool place_ns_supported(uint32_t n_nodes, uint32_t n_domains);
int launch_place_ns(const lwse_node_rec* d_nodes, const uint32_t* d_dom_first, const uint32_t* d_node_order, uint32_t n_nodes,
                    uint32_t n_domains, const lwse_place_req* d_reqs, uint32_t n_reqs,
                    const uint32_t* d_occupancy, uint32_t n_parts, uint64_t part_stride_bytes, uint32_t n_namespaces,
                    lwse_place_out* d_out, void* d_scratch, size_t scratch_bytes, bool fresh, uint32_t call_index, bool scan,
                    int sm_count, cudaStream_t s, const uint32_t** d_counters_out, bool first_pdl,
                    const PlaceNsChanges* changes, const PlaceNsExchange* xch, PlaceNsIndex index);
size_t place_ns_scratch_bytes(uint32_t n_nodes, uint32_t n_domains, uint32_t n_reqs, uint32_t n_namespaces);
size_t node_index_scratch_bytes(uint32_t n_domains);
// The index block's scan (one CTA): first[0..n] = the exclusive scan of count[0..n) and its total, cursor = first,
// count back to zero.
int launch_index_scan(uint32_t* d_count, uint32_t* d_first, uint32_t* d_cursor, uint32_t n, cudaStream_t s);
int launch_node_index(const lwse_node_rec* d_nodes, uint32_t n_nodes, uint32_t n_domains, uint32_t* d_dom_first,
                      uint32_t* d_node_order, uint32_t* d_node_pos, void* d_scratch, int sm_count, cudaStream_t s,
                      bool pdl);
int launch_place_whatif_index(const lwse_place_req* d_reqs, uint32_t n_reqs, uint32_t n_namespaces, const uint8_t* d_touched,
                              uint32_t n_nodes, uint32_t n_domains, void* d_scratch, int sm_count, cudaStream_t s);
int launch_place_whatif_diff(const lwse_place_out* d_before, const lwse_place_out* d_after, uint32_t n_resident, uint32_t n_total,
                             uint32_t* d_rows, lwse_place_out* d_outs_before, lwse_place_out* d_outs_after, uint32_t capacity,
                             uint32_t* d_counts, int sm_count, cudaStream_t s);

// ---- lwse_ds_kernels.cu ----
int launch_ds_sweep(const lwse_ds_tables* t, int sm_count, cudaStream_t s);

struct DsTickHost {
  const lwse_ds_out* prev_ds_out;
  const lwse_ds_role_out* prev_role_out;
  const lwse_ds_revrole_out* prev_revrole_out;
  lwse_ds_out* m_ds_out;
  lwse_ds_role_out* m_role_out;
  lwse_ds_revrole_out* m_revrole_out;
  uint8_t* marks;
  uint32_t* rows;
  uint32_t* counters;  // [0] count, [1] ticket
  uint32_t* host_words;
  uint32_t seq;
  bool all;
  const lwse_ds_link* links;  // non-null: the linked instance
  const lwse_lws_rec* lws;
  const lwse_lws_out* lws_out;
  uint32_t n_lws;
};
int launch_ds_tick(const lwse_ds_tables* t, const DsTickHost* h, int sm_count, cudaStream_t s);

struct DsForecastHost {
  lwse_ds_revrole_rec* rows;
  lwse_ds_out* s_ds_out;
  lwse_ds_role_out* s_role_out;
  lwse_ds_revrole_out* s_revrole_out;
  lwse_ds_forecast* fc;
  lwse_ds_forecast_role* fc_role;
  lwse_ds_role_out* steps;  // the write pass's rows (device scratch)
  uint32_t step_capacity;
  bool want_steps;  // a trajectory is asked for: the scan marks what does not fit in step_capacity
  unsigned long long* totals;  // device, 2 words, zeroed by the caller
};
int launch_ds_forecast(const lwse_ds_tables* t, const DsForecastHost* h, bool write_pass, int sm_count, cudaStream_t s);

// DS drain (lwse_resident_ds_drain*): the link table and the baseline LWS rows it points into.
struct DsDrainLink {
  const lwse_ds_link* links;
  const lwse_lws_rec* lws;
  const lwse_lws_out* lws_out;  // the baseline results (ready_before)
  uint32_t n_lws;
};
// A linked DS sweep of t into t's outputs, reading ready counts from `ready_from` (the baseline, or its copy
// with the drain's lost groups taken off) through the link rule of `lk`.
int launch_ds_drain_sweep(const lwse_ds_tables* t, const DsDrainLink* lk, const lwse_lws_out* ready_from, int sm_count,
                          cudaStream_t s);
// The set form's diff: t's outputs (after) against `before`; touched DS appended to rows (up to capacity).
// counts (device, zeroed by the caller): [16] touched (the append cursor) [17] service lost [18] old service
// lost [19] stalled [20] changed [21] rows touched [22] rows zeroed [23] rows linked.
struct DsDrainDiffHost {
  const lwse_ds_out* before_ds_out;
  const lwse_ds_role_out* before_role_out;
  const lwse_ds_revrole_out* before_revrole_out;
  const uint32_t* lost;  // [n_lws]
  lwse_ds_drain* rows;
  uint32_t capacity;
  uint32_t* counts;
};
int launch_ds_drain_diff(const lwse_ds_tables* t, const DsDrainLink* lk, const DsDrainDiffHost* h, int sm_count,
                         cudaStream_t s);
// The reverse link index of the per-key form: LWS row → the revision-role rows that take its value, once per DS
// whose ranges hold the row (DS ranges may overlap).  fill = false: count[L] += rows per L (count zeroed by the
// caller) and *total (u64, zeroed by the caller) += all of them.  fill = true: every such row's entry
// {DS row, slot (0xFF: the new revision) | 0x100 when a spec role, ready_before, 0} at cursor[L]++, written only
// below capacity (entries holds capacity rows; the caller sizes it from *total).
int launch_ds_drain_links(const lwse_ds_tables* t, const DsDrainLink* lk, uint32_t* count, uint32_t* cursor, uint4* entries,
                          uint32_t capacity, unsigned long long* total, bool fill, int sm_count, cudaStream_t s);
constexpr uint32_t kDsDrainNewSlot = 0xFFu;
constexpr uint32_t kDsDrainSpec = 0x100u;

// ---- lwse_lws_forecast_kernels.cu ----
struct LwsForecastHost {
  const lwse_lws_rec* lws;
  uint32_t n_lws;
  const lwse_group_out* group_out;
  uint32_t n_groups;
  unsigned long long* slot_off;  // [n_lws]
  uint8_t* slots;                // n_slots bytes (+ 8), sized after launch_lws_forecast_slots
  uint32_t n_slots;
  lwse_lws_forecast* fc;
  lwse_lws_forecast_step* steps;  // the write pass's rows (device scratch)
  uint32_t steps_rows;            // rows of `steps`
  uint32_t step_capacity;
  bool want_steps;               // a trajectory is asked for: the scan marks what does not fit
  unsigned long long* totals;    // device: [0] rows needed, [1] rows written, [2] slots, [3] refused accesses
                                 // (zeroed by the caller), then forecast_scan_words(n_lws) words for the scans
};
int launch_lws_forecast_slots(const LwsForecastHost* h, int sm_count, cudaStream_t s);
int launch_lws_forecast(const LwsForecastHost* h, bool write_pass, int sm_count, cudaStream_t s);

// ---- lwse_rollout_whatif_kernels.cu ----
struct RolloutWhatifHost {
  const lwse_lws_rec* lws;        // the resident rows
  const lwse_group_rec* groups;   // the resident group rows
  uint32_t n_groups;
  const uint32_t* rows;           // [n] the proposals' resident rows (< n_lws, checked by the engine)
  uint32_t n;
  unsigned long long* off;        // [n] each proposal's first scratch group row (the layout writes them)
  lwse_lws_rec* s_lws;            // [n] the proposed rows; the gather sets group_base / group_count
  lwse_group_rec* s_groups;       // the gathered group rows
  uint32_t* s_src;                // per gathered row: the resident row of a foreign-owned row, else LWSE_NONE
};
// The layout: off[i] = the exclusive prefix of the proposals' gathered rows, *total = their sum (u64).
// sums: forecast_scan_words(n) words.
int launch_rollout_whatif_layout(const RolloutWhatifHost* h, unsigned long long* sums, unsigned long long* total,
                                 cudaStream_t s);
int launch_rollout_whatif_gather(const RolloutWhatifHost* h, int sm_count, cudaStream_t s);
// The foreign-owned rows' baseline results into d_out and the sweep's flag column (lws_sweep_flag_column).
int launch_rollout_whatif_restore(const uint32_t* d_src, const lwse_group_out* d_baseline, lwse_group_out* d_out,
                                  uint8_t* d_gflag8, uint32_t n_rows, int sm_count, cudaStream_t s);

// ---- lwse_ds_whatif_kernels.cu ----
struct DsWhatifHost {
  lwse_ds_tables t;                   // the resident DS tables (inputs only)
  const lwse_ds_link* links;          // the resident link table, [t.n_revroles]
  const lwse_ds_proposal* proposals;  // [n] (ds < t.n_ds and known flags, checked by the engine)
  const lwse_ds_role_rec* q_roles;    // [n * LWSE_DS_MAX_ROLES] the query's role rows, or null when no proposal
                                      // has LWSE_DSP_ROLES
  uint32_t n;
  uint32_t* count;                    // [n] revision-role rows each proposal gathers (the count kernel writes them)
  uint32_t* off;                      // [n] its first scratch revision-role row (the layout writes them)
  lwse_ds_rec* s_ds;                  // [n] the proposed DS rows
  lwse_ds_role_rec* s_roles;          // [n * LWSE_DS_MAX_ROLES] their role rows, proposal i's at i * 10
  lwse_ds_revrole_rec* s_revroles;    // the gathered revision-role rows ...
  lwse_ds_link* s_links;              // ... and their link rows
};
// The layout: count[i], then off[i] = their exclusive prefix and *total = their sum (u64, < 2^32 for
// n <= LWSE_DS_WHATIF_MAX_PROPOSALS).  sums: forecast_scan_words(n) words.
int launch_ds_whatif_layout(const DsWhatifHost* h, unsigned long long* sums, unsigned long long* total, int sm_count,
                            cudaStream_t s);
int launch_ds_whatif_gather(const DsWhatifHost* h, int sm_count, cudaStream_t s);

// ---- lwse_drain_kernels.cu ----
// The drain what-if's counters (device, 16 words, zeroed by the caller): [0] changed rows [1] pods evicted
// [2] leaders evicted [3] groups restarted [4] ready groups restarted [6..7] pods recreated (u64).
int launch_drain_mark(const uint8_t* d_mask, uint32_t n_nodes, const lwse_pod_ident* d_ident, uint8_t* d_state, uint64_t n_pods,
                      lwse_group_rec* d_groups, uint32_t n_groups, uint32_t* d_counts, int sm_count, cudaStream_t s);
int launch_drain_diff(const lwse_group_out* d_before, const lwse_group_out* d_after, const lwse_group_rec* d_groups,
                      uint32_t n_groups, uint32_t* d_rows, lwse_group_out* d_outs_before, lwse_group_out* d_outs_after,
                      uint32_t capacity, uint32_t* d_counts, int sm_count, cudaStream_t s);
// d_cost: n_nodes rows with `pods` filled in and every other field zero.
int launch_drain_cost(const lwse_lws_rec* d_lws, uint32_t n_lws, const lwse_group_rec* d_groups, uint32_t n_groups,
                      const uint8_t* d_state, const lwse_pod_ident* d_ident, uint64_t n_pods, const lwse_group_out* d_baseline,
                      lwse_drain_cost* d_cost, uint32_t n_nodes, int sm_count, cudaStream_t s);
// The node mask of a set of domains (d_domains: n_domains bytes, 1 = drained) into d_mask (n_nodes bytes).
int launch_drain_domain_mask(const uint8_t* d_domains, uint32_t n_domains, const lwse_node_rec* d_nodes, uint32_t n_nodes,
                             uint8_t* d_mask, int sm_count, cudaStream_t s);
// The drain budget's set form over a what-if sweep (d_after) against the baseline: touched rows appended to
// d_rows (up to capacity); counters [8] touched [9] breached [10] loses available [11] already below.
int launch_drain_budget(const lwse_lws_rec* d_lws, const lwse_lws_out* d_lws_out, uint32_t n_lws, const lwse_group_rec* d_groups,
                        const lwse_group_out* d_before, const lwse_group_out* d_after, uint32_t n_groups,
                        lwse_drain_budget* d_rows, uint32_t capacity, uint32_t* d_counts, int sm_count, cudaStream_t s);
// The drain budget's per-key form.  Pass 0: the key rows (cost zeroed by the caller) get their pods and cost
// totals, and counts[0..1] (u64, zeroed by the caller) the (group, key) pairs the table must hold.  Pass 1
// (keys all-ones and vals zeroed by the caller, table_mask + 1 a power of two > the pairs): the (LWS, key)
// table, then the budget columns of the key rows; counts[2] = inserts the table refused.
struct DrainBudgetCostLaunch {
  const lwse_lws_rec* lws;
  const lwse_lws_out* lws_out;
  const lwse_group_rec* groups;
  const uint8_t* pod_state;
  const lwse_pod_ident* pod_ident;
  const lwse_group_out* baseline;
  const lwse_node_rec* nodes;
  const uint32_t* occupancy;
  lwse_drain_budget_cost* cost;
  unsigned long long* keys;
  uint4* vals;
  uint32_t* counts;
  uint64_t n_pods;
  uint32_t n_lws, n_groups, n_nodes, n_domains, n_keys, table_mask;
  bool by_domain;
};
// Pass 2: the (LWS, key) table alone (pass 1 without the budget columns).
int launch_drain_budget_cost(const DrainBudgetCostLaunch* p, int pass, int sm_count, cudaStream_t s);
// The DS drain's set form: lost[L] (the drain budget's lost groups of every LWS row, d_after a what-if sweep
// against the baseline d_before) and d_lws_after, a copy of d_lws_out with ready_replicas - lost[L].
int launch_ds_drain_lost(const lwse_lws_rec* d_lws, const lwse_lws_out* d_lws_out, uint32_t n_lws, const lwse_group_rec* d_groups,
                         const lwse_group_out* d_before, const lwse_group_out* d_after, uint32_t n_groups, uint32_t* d_lost,
                         lwse_lws_out* d_lws_after, int sm_count, cudaStream_t s);
// The DS drain's per-key form over the drain budget's (LWS, key) table (vals.y = lost(L, key)) and the reverse
// link index.  Pass 0: counts[0..1] (u64, zeroed by the caller) = the (row, key) pairs.  Pass 1 (keys all-ones
// and vals zeroed by the caller, table_mask + 1 a power of two > the pairs): the (DS, key) table, the key rows'
// rows_touched / rows_zeroed, then the DS columns; counts[2] = inserts the table refused.
struct DsDrainCostLaunch {
  const unsigned long long* lws_keys;
  const uint4* lws_vals;
  uint32_t lws_mask;
  const uint32_t* first;  // [n_lws + 1]
  const uint4* entries;
  const lwse_ds_out* before;  // the before sweep's ds_out
  lwse_ds_drain_cost* cost;   // n_keys rows, zeroed by the caller
  unsigned long long* keys;   // the (DS, key) table: DS row << 32 | key
  uint2* vals;                // {bits, old revisions with a zeroed spec row}
  uint32_t table_mask;
  uint32_t* counts;
};
int launch_ds_drain_cost(const DsDrainCostLaunch* p, int pass, int sm_count, cudaStream_t s);

// ---- lwse_drain_place_kernels.cu (and the drain instance of the namespace kernel) ----
// lwse_resident_drain_place_cost.  counts (device, 16 words, zeroed by the caller): [0] PLACED [1] UNSCHEDULABLE
// [2] CONFLICT baseline rows, [3] rule-(b) candidates, [4] items, [5] refused item inserts, [6] restart pairs.
struct DrainPlaceLaunch {
  const lwse_node_rec* nodes;
  const uint32_t* occupancy;
  const uint32_t* dom_first;           // the node index every placement form reads
  const uint32_t* node_order;
  uint32_t* dom_free;                  // [n_domains] free slots per domain (pass 0 writes them)
  const lwse_place_req* reqs;
  const lwse_place_out* base;          // the baseline rows
  const lwse_drain_budget_cost* cost;  // the drain budget's pass 0 rows: groups_restarted per key
  uint32_t n_nodes, n_domains, n_reqs, n_namespaces, n_groups, n_keys;
  bool by_domain;
  const unsigned long long* pairs;     // restart pairs key << 32 | group
  uint32_t n_pairs;
  uint32_t* g_count;                   // [n_groups] pinned request rows per group (zero between calls)
  uint32_t* g_first;                   // [n_groups + 1]
  uint32_t* g_cursor;                  // [n_groups]
  uint32_t* g_reqs;                    // [n_reqs]
  uint32_t* u_count;                   // [n_keys] |U_k| (zero between calls)
  uint32_t* u_first;                   // [n_keys + 1]
  uint32_t* u_cursor;                  // [n_keys]
  uint32_t* u_rows;                    // [n_unpinned]
  uint32_t n_unpinned;                 // u_first[n_keys], once pass 1 is done
  uint32_t* pos;                       // [n_reqs] request row -> position in the namespace index
  unsigned long long* item_keys;       // the (key, namespace) set: key << 32 | namespace, all-ones when free
  uint32_t item_mask;
  uint2* items;
  uint32_t item_capacity;
  lwse_drain_place_cost* rows;         // [n_keys]
  uint32_t* counts;
  // the solve
  void* round;                         // namespace-form scratch (place_ns_scratch_bytes) holding the index of every namespace
  size_t round_bytes;
  lwse_place_out* s_out;               // [grid * slice_rows]
  uint32_t* s_unpinned;                // [grid * slice_rows]
  uint8_t* s_marks;                    // [grid * slice_rows]
  uint32_t slice_rows, grid;
};
// Pass 0 (after the namespace index and the drain budget's pass 0): free slots per domain, the baseline totals, the group -> pinned
// request index (count, scan, fill), U_k's leader rows counted, the rule-(b) candidates counted.
// Pass 1 (pairs written): U_k's rows of restarted groups counted, then the U_k index scanned.
// Pass 2 (u_rows, items sized): U_k filled, the key rows started, the items gathered (and the rows of U_k
// outside every namespace counted), then the solve.
int launch_drain_place(const DrainPlaceLaunch* p, int pass, int sm_count, cudaStream_t s);
// The drain budget walk in pair mode: every restart pair key << 32 | group into pairs[p->counts[8]++] (below capacity).
int launch_drain_restart_pairs(const DrainBudgetCostLaunch* p, unsigned long long* pairs, uint32_t capacity, int sm_count,
                               cudaStream_t s);
int launch_place_ns_drain(const DrainPlaceLaunch* p, int sm_count, cudaStream_t s);

// ---- lwse_rollout_place_kernels.cu ----
// Rollout placement (lwse_resident_rollout_place).  Entry i: resident row rows[i], namespace ns[i], proposal
// recs[i] (null: the resident row), forecast row fc[fc_by_row ? rows[i] : i].
struct RolloutPlaceLaunch {
  const lwse_lws_rec* lws;        // the resident rows
  const lwse_group_rec* groups;   // the resident group rows
  uint32_t n_groups;
  const uint32_t* rows;           // [n]
  const uint32_t* ns;             // [n]
  const lwse_lws_rec* recs;       // [n] or null
  const lwse_lws_forecast* fc;
  bool fc_by_row;
  uint32_t n;
  uint32_t* rows_out;             // [n] lwse_rollout_place, 16 words each
  uint4* ent;                     // [n] {first extra row, |E_i|, group_base, group_count}
  uint32_t* e_count;              // [n] |E_i| (zero between calls: the scan clears it)
  uint32_t* e_first;              // [n + 1]
  uint32_t* e_cursor;             // [n]
  uint2* items;                   // [n] {entry, namespace}: answerable entries with E_i non-empty
  uint32_t* counts;               // 32 words, zeroed by the caller: [0] items [1] max |E_i| [2..3] sum |E_i| (u64),
                                  // [4..9] the finish's totals, [16..22] a place_whatif_diff block over the baseline
                                  // alone (its PLACED / UNSCHEDULABLE / CONFLICT at [20..22])
  lwse_place_req* extra;          // [sum |E_i|]
  // the solve
  const lwse_node_rec* nodes;
  const uint32_t* occupancy;
  const uint32_t* dom_first;
  const uint32_t* node_order;
  const lwse_place_req* reqs;     // the resident request rows
  const lwse_place_out* base;     // the baseline rows
  uint32_t n_nodes, n_domains, n_reqs, n_namespaces;
  void* round;                    // namespace-form scratch holding the index of every namespace
  size_t round_bytes;
  lwse_place_out* s_out;          // [grid * slice_rows]
  uint32_t* s_unpinned;           // [grid * slice_rows]
  uint32_t slice_rows, grid;
};
// Pass 0: the count kernel (flags, |E_i|, the rows started, the items).  Pass 1 (after the host read max |E_i|):
// the scan, the fill of the extra rows, the capacities and the solve, then the finish.
int launch_rollout_place(const RolloutPlaceLaunch* p, int pass, int sm_count, cudaStream_t s);
int launch_place_ns_rollout(const RolloutPlaceLaunch* p, int sm_count, cudaStream_t s);

// ---- lwse_rollout_place_wave_kernels.cu ----
// Rollout placement waves (lwse_resident_rollout_place_waves), over the rollout placement's setup p (its rows are
// the alone rows).  A key takes part when it is SOLVED and clean alone; the K_ns keys of a namespace take rounds
// 0 .. K_ns - 1 in query order.  Slot s = ns_first[ns] + w holds column (ns, w): its list of entries (at
// ns_first[ns] * wc + w * K_ns in col), its extra rows, its committed contribution and the probe row of the round.
struct RolloutPlaceWavesLaunch {
  RolloutPlaceLaunch p;
  uint32_t constraints, max_waves;
  uint32_t wc;                    // list stride: min(max_waves, R)
  uint32_t* st;                   // 16 words, zeroed: [0] round [1] items [2] R [3] max T_ns [4] active namespaces
  uint32_t* rank;                 // [n] the key's round, LWSE_NONE when it does not take part
  uint32_t* ns_count;             // [n_ns] K_ns (the scan zeroes it)
  uint32_t* ns_first;             // [n_ns + 1]
  uint32_t* ns_cursor;            // [n_ns]
  uint32_t* ns_extra;             // [n_ns] T_ns, the extra rows of the namespace's keys, zeroed
  uint32_t* ns_open;              // [n_ns] p_ns, the waves the namespace's keys use, zeroed
  uint32_t* ns_keys;              // [n] per namespace its keys in query order
  uint32_t* act;                  // [n] the namespaces with a key
  uint4* desc;                    // [n] per slot: {k, first list entry, list length, column rows}
  uint4* col;                     // [n * wc] {E_j's first extra row, offset in the column, group_base, group_count}
  uint32_t* col_n;                // [n] per slot: list length, zeroed
  uint32_t* col_rows;             // [n] per slot: the column's extra rows, zeroed
  uint32_t* contrib;              // [n * 11] per slot: the committed contribution, zeroed
  uint32_t* res;                  // [n * 16] per slot: the round's probe row (words 4..15 as lwse_rollout_place's)
  uint2* items;                   // [n] {slot, namespace}
  uint32_t* wtot;                 // [64 * 16] per wave: n_keys, the 11 counters, namespaces; zeroed
  uint8_t* out;                   // the answer: 8 words of totals, n lwse_rollout_wave_key, 64 lwse_rollout_wave
  lwse_place_out* s_out;          // [grid * slice_rows]
  uint32_t* s_unpinned;           // [grid * slice_rows]
  uint32_t slice_rows, grid;      // (grid 0: no column holds an extra row; no solve)
};
// Pass 0 (after the setup's finish): the key rows, the ranks, the scan and the per-namespace key lists.  Pass 1
// (captured, replayed R times): items, the wave instance of place_ns_kernel, commit.  Pass 2: the finish.
int launch_rollout_place_waves(const RolloutPlaceWavesLaunch* w, int pass, int sm_count, cudaStream_t s);
int launch_place_ns_rollout_wave(const RolloutPlaceWavesLaunch* w, cudaStream_t s);

// ---- lwse_scale_headroom_kernels.cu ----
// Scale headroom (lwse_resident_scale_headroom), over the rollout placement's chain p on the resident rows (no
// proposals, fc by row).  Entry i bisects [lo, hi) = st[i].{x, y}; each round's probes are p's rows, solved by
// launch_rollout_place pass 1 as it stands.
struct ScaleHeadroomLaunch {
  RolloutPlaceLaunch p;
  const int32_t* ceilings;        // [n] c_i (negative: none), or null
  uint32_t constraints;           // LWSE_RPW_*
  uint32_t n_domains;             // R_pig's bound (p's solve fields are set only after the setup)
  uint4* st;                      // [n] {lo, hi, the entry's bits, r0}
  const uint32_t* cur;            // [n * 16] p's rows after the setup's solve: the probe at r0 of a settled entry
  uint32_t* clean;                // [n * 16] the row of the highest clean probe above r0
  uint32_t* trig;                 // [n * 16] the row of the lowest triggering probe
  uint32_t* words;                // 8 words, zeroed: [0] entries that search [1] max |E| [2..3] sum |E| (u64) [4] rounds
  uint32_t* out;                  // the answer: 8 words of totals (zeroed), then n lwse_scale_headroom
};
// Pass 0 (after rollout_place pass 0): the setup kernel.  Pass 1 (captured, replayed words[4] times, after the
// setup's solve and the copy of its rows to cur): the round kernel, launch_rollout_place pass 1, the commit.
// Pass 2: the finish.
int launch_scale_headroom(const ScaleHeadroomLaunch* h, int pass, int sm_count, cudaStream_t s);

// ---- lwse_place_explain_kernels.cu ----
// lwse_resident_place_explain over one round: its node, request and result rows (the baseline's in place, or a
// what-if round's scratch) and the resident occupancy.
struct PlaceExplainLaunch {
  const lwse_node_rec* nodes;        // [n_nodes]
  const uint32_t* occupancy;         // [n_nodes] or null
  const lwse_place_req* reqs;        // [n_rows]
  const lwse_place_out* res;         // [n_rows]
  uint32_t n_nodes, n_domains, n_rows, n_namespaces;
  bool by_mask;                      // select the rows whose result flags share a bit with `mask` into `list`
  uint32_t mask;
  uint32_t* chunk_count;             // by mask: [n_chunks] (256 rows each), then the scan's first [n_chunks + 1]
  uint32_t* chunk_first;             //   and cursor [n_chunks]
  uint32_t* chunk_cursor;
  uint32_t* list;                    // the listed rows: filled by mask, or the caller's (uploaded)
  const uint32_t* n_list;            // device word: the rows listed (by mask: chunk_first[n_chunks])
  uint32_t n_listed;                 // their bound, for the grids (by mask: n_rows)
  uint32_t* dom;                     // [3 * n_domains] dom_free | usable | free_all, zeroed by the caller
  uint8_t* ns_mark;                  // [n_namespaces] namespaces of the listed rows, zeroed by the caller
  unsigned long long* tkeys;         // [table_mask + 1] the holder table: ns << 32 | d, all-ones when free ...
  unsigned long long* tvals;         // ... and the holder's spec key (all-ones before)
  uint32_t table_mask;
  lwse_place_explain_row* out;       // [capacity]
  uint32_t capacity;
  unsigned long long* totals;        // 16 words, zeroed by the caller: [0..7] the class sums, [8..14] the flag counts
};
// The stats, the selection (count, scan, fill by mask; mark by list), the holder table, the explanation.
int launch_place_explain(const PlaceExplainLaunch* p, int sm_count, cudaStream_t s);

// ---- lwse_drain_wave_kernels.cu ----
// lwse_resident_drain_waves.  out: the query totals (16 B), m lwse_drain_wave_key rows, then max_waves
// lwse_drain_wave rows (the opened ones written).  counts (device, u64, zeroed by the caller): [0] the restart pairs
// of every key, [1] pairs the key buckets refused.
struct DrainWavesLaunch {
  const lwse_lws_rec* lws;
  const lwse_lws_out* lws_out;
  const lwse_group_rec* groups;
  const lwse_group_out* baseline;
  const lwse_drain_budget_cost* cost;  // the drain budget's pass 0 rows of every key
  const uint32_t* ids;                 // [m] the query's keys
  uint32_t* pos_of;                    // [n_keys] the position of a listed key; all-ones (set by the caller) otherwise
  uint32_t* count;                     // [m] the key buckets: pairs per position (zero between calls)
  uint32_t* first;                     // [m + 1]
  uint32_t* cursor;                    // [m]
  const unsigned long long* pairs;     // the pair walk's key << 32 | group
  uint32_t n_pairs;
  uint4* recs;                         // [first[m]] {group, owner, bits, pod_count} by position
  uint32_t* l_count;                   // [n_lws] 1 for a touched LWS row (zero between calls)
  uint32_t* l_first;                   // [n_lws + 1] its dense row
  uint32_t* l_cursor;                  // [n_lws]
  uint4* dense;                        // [n_lws] {ready_before, floor, flags, 0} by dense row
  uint32_t n_dense;                    // l_first[n_lws], once pass 1 is done
  uint32_t* lost;                      // [n_dense * cols] lost groups per (dense row, wave), zeroed by the caller
  uint32_t cols;                       // min(max_waves, m) + 1: the waves and the key-alone column
  unsigned long long* g_waves;         // [n_groups] the waves that hold the group, zeroed by the caller
  unsigned long long* row_waves;       // [2 * n_dense] the waves touching the row / losing one of its groups below replicas
  uint32_t* stamps;                    // [2 * n_dense] the last position that touched / breached the row alone, zeroed
  uint8_t* out;
  unsigned long long* counts;
  uint32_t n_lws, n_groups, n_keys, m, max_waves;
};
// Pass 0 (after the drain budget's pass 0): positions, bucket sizes and the alone columns; the buckets scanned.
// Pass 1 (pairs written): the buckets filled, the touched rows scanned, the dense rows.  Pass 2 (n_dense, lost and
// the wave masks sized): the plan, then the wave rows' per-row columns and pods / leaders.
int launch_drain_waves(const DrainWavesLaunch* p, int pass, int sm_count, cudaStream_t s);
// lwse_resident_ds_drain_waves: passes 1 and 2 of launch_drain_waves with the DS caps.  caps[n_lws] (device) holds
// per LWS row kCapLinked and the LWSE_DSW_DS_* bits of the gated rows linked to it (ds_drain_waves_caps).  Pass 1
// binds the ready member pairs of evaluated or linked rows and writes each dense row's slack under `constraints`;
// pass 2 runs the plan against those slacks, then the wave rows' per-row columns.
constexpr uint32_t kCapLinked = 1u << 4;
int launch_drain_waves_capped(const DrainWavesLaunch* p, const uint32_t* caps, uint32_t constraints, int pass, int sm_count,
                              cudaStream_t s);

// The drain waves finish alone (the wave rows' per-row columns and pods / leaders), after a plan written elsewhere.
int launch_drain_waves_finish(const DrainWavesLaunch* p, int sm_count, cudaStream_t s);

// ---- lwse_drain_place_wave_kernels.cu (and the set-overlay instance of the namespace kernel) ----
// lwse_resident_drain_place_waves.  The step state lives in device memory so that one captured step replays for
// every key: the key and its position, the open waves, the step's items and refusals, the floor verdicts of the
// columns, the status counts.
struct DpwState {
  uint32_t key, i, n_open, n_items, refused, alone_bad, touched, breached;
  unsigned long long bad;  // the open waves whose floor the key breaks
  uint32_t status[4];
};
struct DrainPlaceWavesLaunch {
  DrainWavesLaunch w;              // the floor plan (the drain waves chain up to its dense rows)
  DrainPlaceLaunch p;              // the drain placement after its passes: U_k, positions, dom_free, the alone rows
  DpwState* st;
  uint32_t constraints, max_waves;
  unsigned long long* u_wave;      // [n_reqs] bit w: the row is in U of wave w
  unsigned long long* key_wave;    // [n_keys] bit w: the node (domain) is in wave w
  unsigned long long* ns_wave;     // [n_namespaces] bit w: the namespace is solved for wave w
  uint32_t* drained;               // [64 * n_domains] node scope: the free slots wave w drains from domain d
  uint32_t* wnons;                 // [64 * 16] per wave: [1] |U_W|, [2..10] its rows of no namespace counted
  uint32_t* wplace;                // [64 * 16] per wave: its last probe's counts (lwse_drain_place_cost words)
  uint32_t* col_rows;              // [64 * 16] the step's column rows (lwse_drain_place_cost words)
  uint32_t* col_ns;                // [64 * n_namespaces] the step's (column, namespace) flags
  uint2* items;                    // {column, namespace}
  uint32_t item_capacity;
  uint32_t* dix_count;             // [n_domains] the rule-(b) rows by baseline domain (count | first | cursor)
  uint32_t* dix_first;
  uint32_t* dix_cursor;
  uint32_t* dix_rows;              // [n_reqs]
  uint32_t* kalone;                // [m] the LWSE_DPW_* bits each key triggers alone
  uint32_t* wbreach;               // [64] lws_breached per wave
  uint8_t* out;                    // the answer: totals (16 B), m key rows, max_waves wave rows
};
// Pass 0: the domain index and the first columns.  Pass 1: one step.  Pass 2: the finish.
int launch_drain_place_waves(const DrainPlaceWavesLaunch* d, int pass, int sm_count, cudaStream_t s);
int launch_place_ns_drain_set(const DrainPlaceWavesLaunch* d, int sm_count, cudaStream_t s);

// ---- lwse_ds_drain_wave_kernels.cu ----
// lwse_resident_ds_drain_waves, around the drain waves chain.  Pass 0 (after the before sweep into t's outputs):
// caps[L] |= the bits of every row the sweep reads that takes L's value (caps zeroed by the caller).  Pass 1 (after
// launch_drain_waves_capped pass 2 and the DS per-key form): the answer in `out` — the query totals (16 B), m
// lwse_ds_drain_wave_key rows, max_waves lwse_ds_drain_wave rows (zeroed by the caller) — from the plan's rows in
// w.out, the key rows of both per-key forms, each dense row's lost groups per wave and each DS's linked rows.
struct DsDrainWavesLaunch {
  lwse_ds_tables t;                   // the resident DS tables, ds_out = the before sweep
  DsDrainLink lk;
  uint32_t* caps;                     // [n_lws]
  const lwse_ds_drain_cost* ds_cost;  // the DS per-key form's rows of every key
  uint8_t* out;
  uint32_t max_waves;
};
int launch_ds_drain_waves(const DsDrainWavesLaunch* d, const DrainWavesLaunch* w, int pass, int sm_count, cudaStream_t s);

// ---- lwse_sha1_kernels.cu ----
int launch_sha1(const uint8_t* d_bytes, const uint32_t* d_offsets, uint32_t n, uint8_t* d_digests,
                int sm_count, cudaStream_t s);
int launch_subgroup_keys(const uint8_t* d_bytes, const uint32_t* d_offsets, uint32_t n, const int32_t* d_pod_count,
                         const int32_t* d_subgroup_size, const int32_t* d_worker_index, int32_t* d_index_out,
                         uint8_t* d_digests, int sm_count, cudaStream_t s);

// ---- lwse_exchange_kernels.cu ----
int launch_exchange_push(const void* d_local_part, uint8_t* const* d_peer_base, void* d_local_base,
                         uint64_t part_bytes, uint64_t part_stride, uint64_t half_bytes, uint64_t flags_offset,
                         uint64_t step, uint64_t wait_step, uint32_t world, uint32_t rank, cudaStream_t s,
                         bool lagged);

}  // namespace lwse
