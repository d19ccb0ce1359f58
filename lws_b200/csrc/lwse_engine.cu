// C-ABI implementation of include/lwse.h: engine lifecycle, device staging,
// host- and device-pointer entry points.  No CPU compute path exists in this
// library: every sweep is a CUDA kernel launch or the call fails.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <unordered_map>
#include <vector>
#include <new>

#include "lwse_device.cuh"
#include "lwse_launch.cuh"

namespace {

// The CUDA objects all engines hold (allocations, streams, events, graph executables, peer mappings): the owners
// below count each one they acquire and release (lwse_debug_cuda_objects).
std::atomic<int64_t> g_cuda_objects{0};

// A device buffer that only grows (sweeps reuse their staging memory).
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    release();
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) {
      cap = want;
      ++g_cuda_objects;
    } else {
      p = nullptr;
    }
    return e;
  }
  void release() {
    if (p) {
      cudaFree(p);
      --g_cuda_objects;
    }
    p = nullptr;
    cap = 0;
  }
};

// Pinned, mapped host memory that only grows: the host writes / reads it in place and the GPU
// reaches it through `d` (patch arena, change lists, tick words).
struct PinBuf {
  void* h = nullptr;
  void* d = nullptr;
  size_t cap = 0;
  PinBuf() = default;
  PinBuf(const PinBuf&) = delete;
  PinBuf& operator=(const PinBuf&) = delete;
  ~PinBuf() { release(); }
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    release();
    const size_t want = bytes + bytes / 8 + 4096;
    cudaError_t e = cudaHostAlloc(&h, want, cudaHostAllocMapped);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer(&d, h, 0);
    if (e == cudaSuccess) {
      cap = want;
      ++g_cuda_objects;
      memset(h, 0, want);  // sequence words and counters start at zero
    } else if (h) {
      cudaFreeHost(h);
      h = d = nullptr;
    }
    return e;
  }
  void release() {
    if (h) {
      cudaFreeHost(h);
      --g_cuda_objects;
    }
    h = d = nullptr;
    cap = 0;
  }
  bool holds(const void* ptr, size_t bytes) const {
    const uintptr_t a = reinterpret_cast<uintptr_t>(ptr), b = reinterpret_cast<uintptr_t>(h);
    return h && a >= b && a + bytes <= b + cap;
  }
  template <typename T>
  T* dev_of(const T* host_ptr) const {
    return reinterpret_cast<T*>(static_cast<uint8_t*>(d) + (reinterpret_cast<const uint8_t*>(host_ptr) - static_cast<uint8_t*>(h)));
  }
};

// A CUDA handle that destroys itself.  It converts to the raw handle, so it passes wherever one is taken.
template <typename T, cudaError_t (*Destroy)(T)>
struct Owned {
  T h = nullptr;
  Owned() = default;
  Owned(const Owned&) = delete;
  Owned& operator=(const Owned&) = delete;
  ~Owned() { reset(); }
  operator T() const { return h; }
  void reset() {
    if (h) {
      Destroy(h);
      --g_cuda_objects;
    }
    h = nullptr;
  }

 protected:
  cudaError_t adopt(cudaError_t e) {  // the result of the call that created h
    if (e == cudaSuccess)
      ++g_cuda_objects;
    else
      h = nullptr;
    return e;
  }
};

struct Stream : Owned<cudaStream_t, cudaStreamDestroy> {
  // `highest`: at the device's highest stream priority
  cudaError_t ensure(unsigned flags, bool highest = false) {
    if (h) return cudaSuccess;
    if (!highest) return adopt(cudaStreamCreateWithFlags(&h, flags));
    int least = 0, greatest = 0;
    const cudaError_t e = cudaDeviceGetStreamPriorityRange(&least, &greatest);
    return e != cudaSuccess ? e : adopt(cudaStreamCreateWithPriority(&h, flags, greatest));
  }
};

struct Event : Owned<cudaEvent_t, cudaEventDestroy> {
  cudaError_t ensure(unsigned flags) { return h ? cudaSuccess : adopt(cudaEventCreateWithFlags(&h, flags)); }
};

struct GraphExec : Owned<cudaGraphExec_t, cudaGraphExecDestroy> {
  cudaError_t ensure(cudaGraph_t graph) { return h ? cudaSuccess : adopt(cudaGraphInstantiate(&h, graph, 0)); }
};

// The exchange buffers of the peers, by rank (lwse_exchange_connect).  The own rank's entry is the engine's own
// buffer: it is not opened here and never closed.
struct PeerMaps {
  void* p[LWSE_MAX_RANKS] = {};
  bool opened[LWSE_MAX_RANKS] = {};
  PeerMaps() = default;
  PeerMaps(const PeerMaps&) = delete;
  PeerMaps& operator=(const PeerMaps&) = delete;
  ~PeerMaps() { close(); }
  cudaError_t open(uint32_t rank, const cudaIpcMemHandle_t& handle) {
    const cudaError_t e = cudaIpcOpenMemHandle(&p[rank], handle, cudaIpcMemLazyEnablePeerAccess);
    if (e == cudaSuccess) {
      opened[rank] = true;
      ++g_cuda_objects;
    }
    return e;
  }
  void close() {
    for (uint32_t r = 0; r < LWSE_MAX_RANKS; r++) {
      if (opened[r]) {
        cudaIpcCloseMemHandle(p[r]);
        --g_cuda_objects;
      }
      opened[r] = false;
      p[r] = nullptr;
    }
  }
};

// What the placement branch of a tick decided when it was enqueued; a tick graph keeps it for its replays.
struct TickPlaceResult {
  bool place_ns = false;                 // the round runs the namespace kernels (counters in the slot's block)
  const uint32_t* rounds_ptr = nullptr;  // device: where the round counts
};

}  // namespace

struct lwse_engine {
  int device = 0;
  int sm_count = lwse::kSmCount;
  Stream stream;
  Stream side_stream;                  // placement round of lwse_reconcile_device
  Stream hist_stream;                  // copies the unpinned-request count of a round to the host, off the critical path
  Event ev_hist;
  Event ev_fork, ev_join;
  std::mutex mu;
  int last_cuda_error = 0;
  uint64_t launches = 0;
  // resident node table
  DevBuf nodes;
  DevBuf dom_first, node_order, node_pos;  // domain-sorted index of the usable nodes (placement), built on the device
  DevBuf node_ix;                          // its build's per-domain counters and cursors (zero between builds)
  uint32_t n_nodes = 0, n_domains = 0;
  std::vector<lwse_node_rec> h_nodes;      // host mirror of the node table: decides whether a patch needs a new index
  bool node_index_stale = false;           // node patches changed usability / domains since the last build
  bool main_unforked = false;              // a tick without a round patched tables on the engine's stream, and no
                                           // round on the side stream has been ordered behind that scatter yet
  lwse_node_info last_node_info{};         // lwse_resident_node_info
  // staging for the *_host entry points
  DevBuf lws, groups, pod_state, pod_ident, lws_out, group_out, occupancy, scan_scratch;
  DevBuf place_reqs, place_out, place_occ, place_scratch;
  uint64_t ident_rows = ~0ull;       // rows of the identity column resident from the last host sweep
  uint64_t ident_hint_pods = ~0ull;  // n_pods the hint below was measured on
  uint32_t ident_hint_events = 0;    // event pods the previous host sweep of that table visited
  // resident tables (lwse_resident_*)
  DevBuf r_lws, r_groups, r_pst, r_pid, r_lws_out, r_group_out, r_scan;
  DevBuf r_counts;                   // per tick slot (16 words): [0] lws changes, [1] group changes, [2] publish ticket, [4] place changes
  DevBuf r_occ;                      // scheduled pods per node of the resident identity column
  DevBuf r_preq, r_pout, r_pout_prev;  // resident placement requests / results of this and the previous tick
  PinBuf arena;                      // patch arena handed to the caller
  PinBuf stage;                      // staging for patch segments that lie outside the arena
  DevBuf arena_mirror, stage_mirror; // device copies of the two: a tick with many patches moves them with one DMA
                                     // copy per buffer (SM reads of host memory are latency-bound)
  PinBuf chg;                        // change lists: [lws rows | lws out | group rows | group out | place rows | place out]
  DevBuf chg_dev;                    // the same layout in device memory: the kernels append here, a publish kernel copies out
  uint32_t last_changed[2] = {0, 0}; // rows the previous tick reported (sweep lists, placement list): sizes the publish grid
  PinBuf tickw;                      // [0] lws changes [1] group changes [2] place changes [3] placement rounds [4] sequence word
  size_t chg_off[6] = {};
  uint32_t rn_lws = 0, rn_groups = 0, rn_reqs = 0, rn_namespaces = 0;
  uint64_t rn_pods = 0;
  bool r_loaded = false, r_place_loaded = false;
  uint32_t tick_seq = 0;
  // ticks in flight (lwse_resident_tick_submit / _wait): two slots of pinned change lists and words
  struct TickSlot {
    uint32_t seq = 0;
    bool do_sweep = false, do_place = false, published = false, wrote = false;
  } tslot[2];
  uint64_t t_submitted = 0, t_waited = 0;
  size_t chg_bytes = 0;              // one slot of `chg`
  // a tick replayed as a CUDA graph (one cudaGraphLaunch instead of ~10 launches)
  struct TickGraph {
    GraphExec exec;
    uint32_t seen = 0;      // eager ticks with this key so far (the first one lets every buffer settle)
    uint32_t kernels = 0;   // kernel nodes (launch accounting)
    bool failed = false;    // capture or instantiation failed once: this key stays eager
    TickPlaceResult place;  // of the captured placement branch
  };
  std::unordered_map<uint32_t, TickGraph> tick_graphs;
  PinBuf tdesc;                      // 2 slots x kScatterDescBytes: the scatter's segment descriptors of the tick of that parity
  DevBuf tdesc_dev;                  // device copy (the copy node at the root of a tick graph fills it)
  Stream copy_stream;                  // the patch copy of a replayed tick: overlaps the previous tick's kernels
  Event ev_dma;
  Stream pub_stream;                   // the publish kernels: tick k+1 starts while tick k's changed rows travel to the host
  Event ev_done;                       // behind the last kernel of a tick on the engine's stream (both branches joined)
  Event ev_mid;                        // (graph capture) between the condense and the namespace kernel
  int use_graph = 1;                 // LWSE_TICK_GRAPH: 0 never, 1 when a tick is in flight (default), 2 always
  uint64_t graph_ticks = 0;
  Event ev_pub;                      // behind the previous tick's publish kernel: the next tick's side stream starts there
  PinBuf h_counts;                   // 2 words
  DevBuf h_counts_dev;               // event-pod count of the host entry point's sweep
  uint32_t place_calls = 0;          // selects the scratch half
  uint32_t place_geometry[4] = {0, 0, 0, 0};  // (n_reqs, n_namespaces, nodes, domains) the scratch was laid out for
  Event ev_place;                    // end of the last placement call: the next one (any stream) orders behind it
  bool place_pending = false;
  DevBuf place_ns_scratch;           // namespace-parallel form (grouped request tables)
  uint32_t place_ns_calls = 0;
  uint32_t place_ns_geometry[4] = {0, 0, 0, 0};
  uint32_t n_usable = 0;             // nodes a request can use (schedulable, labelled): length of the sorted index
  const uint32_t* place_rounds_ptr = nullptr;  // device: the round counter of the last placement call
  const uint32_t* place_scans_ptr = nullptr;   // device: its (request, round) search counter (grouped form), or null
  bool r_place_grouped = false;      // the resident request table is grouped by namespace
  std::vector<uint32_t> r_req_ns;    // its namespace column (host copy: patches must not regroup it)
  bool r_ns_index_ok = false;        // the namespace index in place_ns_scratch matches that column
                                     // (ungrouped tables; any other namespace-form call overwrites ns_first)
  lwse_tick_info last_tick_info{};   // what the last submitted tick ran (lwse_resident_tick_info)
  const uint32_t* place_counters = nullptr;  // device: counters / phase stamps of the last placement call
  const uint32_t* place_unpinned = nullptr;  // device: its unpinned-request count
  DevBuf ds, ds_roles, ds_revroles, ds_out, ds_role_out, ds_revrole_out;
  // resident DS tables (lwse_ds_resident_*): their own stream, never ordered with the LWS ticks
  Stream ds_stream;
  DevBuf rd_ds, rd_roles, rd_revroles;
  DevBuf rd_out[2], rd_role_out[2], rd_revrole_out[2];  // output sets, alternating by tick parity
  DevBuf rd_marks, rd_ones;          // DS rows the tick's scatter patched / a column of ones the scatter copies there
  DevBuf rd_counters;                // [0] changed rows, [1] CTA ticket
  PinBuf rd_pin;                     // [words | changed rows | ds_out | role_out | revrole_out] mirrors
  size_t rd_off[4] = {};             // offsets of rows / ds_out / role_out / revrole_out in rd_pin
  PinBuf rd_stage;                   // a tick's segments, staged for one H2D copy
  DevBuf rd_stage_dev;
  uint32_t rdn_ds = 0, rdn_roles = 0, rdn_revroles = 0;
  uint32_t rd_seq = 0, rd_parity = 0;
  bool rd_loaded = false, rd_all = false;
  DevBuf rd_links;                   // LWSE_TABLE_DS_LINKS: revision-role row → resident LWS row
  bool rd_linked = false;            // a link patch arrived since the DS load: ticks run the linked sweep
  Event ev_ds_link;                  // the engine's stream at the start of a linked DS tick
  lwse_ds_tick_info last_ds_info{};  // lwse_ds_resident_tick_info
  // rollout forecast (lwse_ds_forecast_*): a private copy of the revision-role rows, the replay's sweep
  // outputs, the forecast rows and the trajectory; never the DS tick's buffers
  DevBuf fc_rows, fc_ds_out, fc_role_out, fc_revrole_out, fc_ds, fc_roles, fc_steps, fc_totals;
  PinBuf fc_words;                   // the two totals, copied back
  bool r_swept = false;              // r_lws_out holds the results of the resident LWS rows: a sweep was enqueued
                                     // since lwse_resident_load and since any LWS-row patch without a sweep
  bool r_groups_swept = false;       // r_group_out holds the results of the resident rows: as r_swept, for
                                     // patches of LWS, group and pod rows
  // rolling-update forecast (lwse_lws_forecast_*): a snapshot of the LWS rows and group results, the private
  // flag slots, the forecast rows and the trajectory, on a stream of its own; never a tick's buffers
  Stream lf_stream;
  Event ev_lf;                       // the engine's stream where a resident forecast takes its snapshot
  DevBuf lf_lws, lf_group_out, lf_slot_off, lf_slots, lf_fc, lf_steps, lf_totals;
  PinBuf lf_words;                   // the three totals, copied back
  // rollout what-if (lwse_resident_rollout_whatif): on lf_stream, the proposals' rows and their resident rows, the
  // layout's offsets and block sums, the gathered group rows with their foreign-row record, the sweep's results
  // and scratch; the forecast that follows uses the lf_* scratch above
  DevBuf rw_rows, rw_lws, rw_off, rw_sums, rw_groups, rw_src, rw_group_out, rw_now, rw_scan;
  bool r_place_current = false;      // r_pout holds the round of the resident node, request and identity rows: a
                                     // tick with LWSE_TICK_PLACE was submitted since lwse_resident_place_load and
                                     // since any patch of those rows made without a round
  // placement what-if (lwse_resident_place_whatif): patched copies of the node and request rows, the what-if
  // round's rows, its own node index and round scratch, on a stream of its own; never a tick's buffers
  Stream wf_stream;
  Event ev_wf;                       // the engine's stream where a what-if takes its snapshot
  Event ev_wf_t0, ev_wf_t1;          // (LWSE_WHATIF_TIMING=1) around the last what-if's device work
  bool wf_timed = false;
  DevBuf wf_nodes, wf_reqs, wf_out, wf_dom_first, wf_node_order, wf_node_pos, wf_node_ix, wf_touched, wf_round, wf_list;
  PinBuf wf_stage;                   // the call's segments, extra rows and namespace mask (the scatter reads them here)
  PinBuf wf_words;                   // the counts, copied back
  uint32_t wf_geometry[4] = {0, 0, 0, 0};  // (n_reqs, n_namespaces, nodes, domains) the round scratch was laid out for
  uint32_t wf_calls = 0;
  // drain what-if / drain cost (lwse_resident_drain_*): on the what-if stream, copies of the state column and the
  // group rows, the sweep's bitmaps and group rows, the node mask, the change list and the cost rows
  DevBuf dr_state, dr_groups, dr_out, dr_scan, dr_mask, dr_list, dr_cost;
  // drain budget (lwse_resident_drain_budget*): the domain mask, the touched rows, the key rows, the (LWS, key)
  // table and its counters
  DevBuf dr_domains, dr_brows, dr_bcost, dr_table, dr_bwords;
  // drain placement (lwse_resident_drain_place_cost): the drain budget's key rows and walk counters, the counters,
  // the free slots per domain, the group -> request and key -> U_k indexes, the restart pairs, U_k's rows, the row
  // positions, the item table and list, the key rows, the all-namespaces mask, the round scratch, the solve's
  // per-CTA slices
  DevBuf dp_cost, dp_words, dp_domfree, dp_gidx, dp_uidx, dp_pairs, dp_urows, dp_pos, dp_items, dp_rows, dp_touched, dp_round,
      dp_slices;
  // rollout placement (lwse_resident_rollout_place): the entries' rows and namespaces, the answer rows, the entries'
  // {first extra row, |E_i|, group range}, the |E_i| index (count | first | cursor), the items, the counters, the
  // extra rows, the all-namespaces mask, the round scratch, the solve's per-CTA slices
  DevBuf rp_in, rp_rows, rp_ent, rp_idx, rp_items, rp_words, rp_extra, rp_touched, rp_round, rp_slices;
  // rollout placement waves (lwse_resident_rollout_place_waves): the round state and wave totals, the per-namespace
  // counts (K_ns | first | cursor | T_ns | p_ns), the per-key ranks, lists and active namespaces, the per-slot
  // state, the column lists, the round's slices, the answer; the answer going back (host)
  DevBuf rq_state, rq_ns, rq_keys, rq_slots, rq_col, rq_slices, rq_out;
  PinBuf rq_host;
  // scale headroom (lwse_resident_scale_headroom): the ceilings, the bounds per entry, the current / clean /
  // triggering rows, the answer (its totals first, the setup's words after the rows); the answer going back (host)
  DevBuf sh_ceil, sh_state, sh_rows, sh_out;
  PinBuf sh_host;
  // placement explanation (lwse_resident_place_explain): on the what-if stream, the selected rows (their count, the
  // mask form's chunk index, the list), the per-domain stats, the namespace marks, the holder table, the totals and
  // rows; the caller's rows going in and the answer's words coming back through px_host
  DevBuf px_sel, px_dom, px_mark, px_table, px_out;
  PinBuf px_host;
  // drain waves (lwse_resident_drain_waves): the drain budget's key rows, the counters, the ids, the key positions, the
  // key buckets (count | first | cursor), the restart pairs, the pair records, the touched-row index (count | first |
  // cursor), the dense rows, the lost counters, the group and row wave masks, the stamps, the answer; the ids going
  // in and the answer coming back through dv_host
  DevBuf dv_cost, dv_words, dv_ids, dv_pos, dv_kidx, dv_pairs, dv_recs, dv_lidx, dv_dense, dv_lost, dv_gwaves, dv_rwaves,
      dv_stamps, dv_out;
  PinBuf dv_host;
  // DS drain waves (lwse_resident_ds_drain_waves): the per-LWS-row caps and the answer; the rest is the drain
  // waves' and the DS drain's scratch
  DevBuf dx_caps, dx_out;
  // drain placement waves (lwse_resident_drain_place_waves): the step state, the wave state (U, key and namespace
  // masks, drained slots, per-wave counts), the column state, the items, the rule-(b) domain index, the alone bits,
  // the answer; the rest is the drain waves' and the drain placement's scratch
  DevBuf dq_state, dq_uwave, dq_kwave, dq_nswave, dq_drained, dq_small, dq_colns, dq_items, dq_dix, dq_out;
  // DS drain (lwse_resident_ds_drain*): lost[L] and the after copy of lws_out, the before / after sweep outputs, the
  // touched DS rows, the reverse link index (count | first | cursor) and its entries, the key rows, the (DS, key) table
  DevBuf dd_lost, dd_lws_after, dd_out[2], dd_role_out[2], dd_revrole_out[2], dd_rows, dd_index, dd_entries, dd_cost, dd_table;
  Event ev_dd;                       // the DS stream where a DS drain starts
  // DS rollout what-if (lwse_resident_ds_rollout_whatif): on the what-if stream, the proposals and the query's role
  // rows, the layout's counts, offsets and block sums, the proposed DS, role, revision-role and link rows, and the
  // linked sweep's outputs; the forecast that follows uses the fc_* scratch above
  DevBuf dw_props, dw_qroles, dw_count, dw_off, dw_sums, dw_ds, dw_roles, dw_revroles, dw_links, dw_now, dw_role_out,
      dw_revrole_out;
  PinBuf dw_words;                   // the layout's total, copied back
  uint32_t r_sweep_flags = 0;        // LWSE_SWEEP_GANG of the most recently submitted sweep (r_group_out's flags)
  DevBuf sha_bytes, sha_offsets, sha_digests, sha_ints;
  PinBuf h_rounds;
  // peer exchange of the multi-GPU placement step (lwse_exchange_*)
  DevBuf xch, xch_peers_dev;
  PeerMaps xch_peer;
  uint32_t xch_world = 0, xch_rank = 0, xch_reqs_per_part = 0;
  uint64_t xch_stride = 0, xch_reqs_off = 0, xch_half = 0, xch_flags_off = 0, xch_step = 0;
  bool xch_connected = false;
};

namespace {

int fail_cuda(lwse_engine* e, cudaError_t err) {
  e->last_cuda_error = (int)err;
  (void)cudaGetLastError();  // clear the sticky-free error state
  return err == cudaErrorMemoryAllocation ? LWSE_ERR_OOM : LWSE_ERR_CUDA;
}

// The result of a launcher (the kernels it launched, or its CUDA error negated): counts the kernels, or fails.
int count_launch(lwse_engine* e, int result) {
  if (result < 0) return fail_cuda(e, (cudaError_t)-result);
  e->launches += (uint64_t)result;
  return LWSE_OK;
}

#define LWSE_CUDA(e, call)                                \
  do {                                                    \
    cudaError_t err__ = (call);                           \
    if (err__ != cudaSuccess) return fail_cuda(e, err__); \
  } while (0)

#define LWSE_LAUNCH(e, call)                              \
  do {                                                    \
    const int rc__ = count_launch(e, (call));             \
    if (rc__ != LWSE_OK) return rc__;                     \
  } while (0)

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Tick graphs freeze device pointers and sizes in their kernel nodes: whatever reallocates or
// resizes a resident buffer drops them (the next ticks re-capture).
void invalidate_tick_graphs(lwse_engine* e) { e->tick_graphs.clear(); }

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    int cur = -1;
    cudaGetDevice(&cur);
    if (prev >= 0 && cur != prev) cudaSetDevice(prev);
  }
};

int check_lws_tables(const lwse_lws_tables* t) {
  if (!t) return LWSE_ERR_INVALID_ARG;
  if (t->n_lws && (!t->lws || !t->lws_out)) return LWSE_ERR_INVALID_ARG;
  if (t->n_groups && (!t->groups || !t->group_out)) return LWSE_ERR_INVALID_ARG;
  if (t->n_pods && (!t->pod_state || !t->pod_ident)) return LWSE_ERR_INVALID_ARG;
  if (t->n_pods > 0xFFFFFFFFull) return LWSE_ERR_UNSUPPORTED;  // pod_base / pod_count are 32-bit
  if (!aligned16(t->lws) || !aligned16(t->groups) || !aligned16(t->lws_out) || !aligned16(t->group_out) ||
      !aligned16(t->pod_state) || !aligned16(t->pod_ident))
    return LWSE_ERR_INVALID_ARG;
  return LWSE_OK;
}

}  // namespace

extern "C" {

static int drain_ticks_locked(lwse_engine* e);  // waits for (and drops the results of) every tick in flight
static bool ds_resident_table(const lwse_engine* e, uint32_t which, void** base, uint32_t* rows, uint32_t* row_bytes);

LWSE_API uint32_t lwse_abi_version(void) { return LWSE_ABI_VERSION; }

LWSE_API const char* lwse_strerror(int status) {
  switch (status) {
    case LWSE_OK: return "ok";
    case LWSE_ERR_INVALID_ARG: return "invalid argument (NULL or misaligned table, bad count)";
    case LWSE_ERR_NO_DEVICE: return "no usable CUDA device (this engine has no CPU fallback)";
    case LWSE_ERR_CUDA: return "CUDA call failed (see lwse_last_cuda_error)";
    case LWSE_ERR_OOM: return "device or pinned memory allocation failed";
    case LWSE_ERR_BAD_TABLE: return "a base/count in a record points outside its table";
    case LWSE_ERR_NOT_READY: return "engine not ready for this call (upload the node table first)";
    case LWSE_ERR_UNSUPPORTED: return "unsupported input";
    default: return "unknown lwse status";
  }
}

LWSE_API uint64_t lwse_hash64(const void* bytes, size_t len) {
  const uint8_t* b = static_cast<const uint8_t*>(bytes);
  uint64_t h = 0xCBF29CE484222325ull;
  for (size_t i = 0; i < len; i++) h = (h ^ b[i]) * 0x100000001B3ull;
  return h;
}

LWSE_API uint32_t lwse_shard_of(uint64_t uid_hash, uint32_t n_shards) {
  if (n_shards <= 1) return 0;
  // finalizer of splitmix64 so that weak uid hashes still spread
  uint64_t x = uid_hash;
  x ^= x >> 30;
  x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27;
  x *= 0x94D049BB133111EBull;
  x ^= x >> 31;
  return (uint32_t)(x % n_shards);
}

LWSE_API int lwse_create(const lwse_config* cfg, lwse_engine** out) {
  if (!cfg || !out) return LWSE_ERR_INVALID_ARG;
  *out = nullptr;
  if (cfg->abi_version != LWSE_ABI_VERSION) return LWSE_ERR_INVALID_ARG;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || cfg->device < 0 || cfg->device >= n) {
    (void)cudaGetLastError();
    return LWSE_ERR_NO_DEVICE;
  }
  lwse_engine* e = new (std::nothrow) lwse_engine();
  if (!e) return LWSE_ERR_OOM;
  e->device = cfg->device;
  DeviceGuard guard(e->device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, e->device) != cudaSuccess) {
    delete e;
    return LWSE_ERR_NO_DEVICE;
  }
  if (prop.major != 9 || prop.minor != 0) {  // the kernels are built for sm_90a only
    delete e;
    return LWSE_ERR_NO_DEVICE;
  }
  e->sm_count = prop.multiProcessorCount;
  // The placement round of a tick (side stream) is short and latency-bound; at the highest priority its CTAs
  // take the first SM slots the sweep kernels free instead of queueing behind their blocks.
  if (e->stream.ensure(cudaStreamNonBlocking) != cudaSuccess ||
      e->side_stream.ensure(cudaStreamNonBlocking, /*highest=*/true) != cudaSuccess ||
      e->ev_fork.ensure(cudaEventDisableTiming) != cudaSuccess || e->ev_join.ensure(cudaEventDisableTiming) != cudaSuccess ||
      e->ev_pub.ensure(cudaEventDisableTiming) != cudaSuccess || e->ev_dma.ensure(cudaEventDisableTiming) != cudaSuccess ||
      e->copy_stream.ensure(cudaStreamNonBlocking) != cudaSuccess || e->pub_stream.ensure(cudaStreamNonBlocking) != cudaSuccess ||
      e->ev_done.ensure(cudaEventDisableTiming) != cudaSuccess || e->ev_mid.ensure(cudaEventDisableTiming) != cudaSuccess ||
      e->hist_stream.ensure(cudaStreamNonBlocking) != cudaSuccess || e->ev_hist.ensure(cudaEventDisableTiming) != cudaSuccess ||
      e->ev_place.ensure(cudaEventDisableTiming) != cudaSuccess || e->h_rounds.reserve(64) != cudaSuccess ||
      e->h_counts.reserve(64) != cudaSuccess) {
    (void)cudaGetLastError();
    delete e;
    return LWSE_ERR_CUDA;
  }
  if (e->h_counts_dev.reserve(64) != cudaSuccess) {
    (void)cudaGetLastError();
    delete e;
    return LWSE_ERR_OOM;
  }
  {
    const char* g = getenv("LWSE_TICK_GRAPH");
    e->use_graph = g ? atoi(g) : 1;
  }
  *out = e;
  return LWSE_OK;
}

// The members free themselves when the engine is deleted, with its device current.
LWSE_API void lwse_destroy(lwse_engine* e) {
  if (!e) return;
  DeviceGuard guard(e->device);
  // work in flight writes buffers that are about to be freed (a device synchronize would also wait for other engines)
  const cudaStream_t streams[] = {e->stream,     e->side_stream, e->hist_stream, e->copy_stream,
                                  e->pub_stream, e->ds_stream,   e->lf_stream,   e->wf_stream};
  for (cudaStream_t s : streams)
    if (s) cudaStreamSynchronize(s);
  delete e;
}

LWSE_API int lwse_last_cuda_error(const lwse_engine* e) { return e ? e->last_cuda_error : 0; }
LWSE_API void* lwse_stream(const lwse_engine* e) { return e ? (void*)e->stream : nullptr; }
LWSE_API uint64_t lwse_launch_count(const lwse_engine* e) { return e ? e->launches : 0; }

// A node a placement request can use: schedulable, labelled with the topology key, a domain in range.
static bool node_usable(const lwse_node_rec& nd, uint32_t n_domains) {
  return (nd.flags & LWSE_NODE_SCHEDULABLE) && (nd.flags & LWSE_NODE_HAS_TOPOLOGY) && nd.domain_id < n_domains;
}

// The node-index rule (ticks and what-ifs alike): a patch needs a new domain-sorted index when it changes
// whether the node is usable, or the domain of a usable node.  Capacity-only patches keep the index.
static bool node_patch_moves_index(const lwse_node_rec& old, const lwse_node_rec& now, uint32_t n_domains) {
  const bool was = node_usable(old, n_domains), is = node_usable(now, n_domains);
  return was != is || (is && old.domain_id != now.domain_id);
}

// The domain-sorted node index (dom_first / node_order / node_pos), rebuilt on `s` from the device node
// rows when node patches made it stale.  Called by every placement call in front of its round (in a tick:
// on the side stream, behind the scatter that patched the rows).  `pdl`: the predecessor on `s` is a kernel.
static int build_node_index_locked(lwse_engine* e, cudaStream_t s, bool pdl, bool* built = nullptr) {
  if (built) *built = false;
  if (!e->node_index_stale) return LWSE_OK;
  LWSE_LAUNCH(e, lwse::launch_node_index((const lwse_node_rec*)e->nodes.p, e->n_nodes, e->n_domains, (uint32_t*)e->dom_first.p,
                                         (uint32_t*)e->node_order.p, (uint32_t*)e->node_pos.p, e->node_ix.p, e->sm_count, s,
                                         pdl));
  e->node_index_stale = false;
  if (built) *built = true;
  return LWSE_OK;
}

LWSE_API int lwse_upload_nodes(lwse_engine* e, const lwse_node_rec* nodes, uint32_t n_nodes,
                               uint32_t n_domains) {
  if (!e || (n_nodes && !nodes) || !aligned16(nodes)) return LWSE_ERR_INVALID_ARG;
  if (n_nodes > LWSE_POD_NODE_MAX) return LWSE_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  {
    const int drc = drain_ticks_locked(e);
    if (drc != LWSE_OK) return drc;
    invalidate_tick_graphs(e);
  }
  // every placement call orders behind the previous one (which may still read the index rewritten here)
  if (e->place_pending) LWSE_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_place, 0));
  LWSE_CUDA(e, e->nodes.reserve((size_t)n_nodes * sizeof(lwse_node_rec) + 16));
  LWSE_CUDA(e, e->dom_first.reserve(((size_t)n_domains + 1) * 4 + 16));
  // (padded to whole rows of 256 entries: the namespace-parallel placement kernel stages the index
  // into shared memory with one bulk copy of that size)
  const size_t order_padded = ((size_t)(n_nodes + 255u) / 256u + 1u) * 1024u;
  LWSE_CUDA(e, e->node_order.reserve(order_padded + 16));
  LWSE_CUDA(e, cudaMemsetAsync(e->node_order.p, 0, order_padded, e->stream));
  LWSE_CUDA(e, e->node_pos.reserve((size_t)n_nodes * 4 + 16));
  LWSE_CUDA(e, e->node_ix.reserve(lwse::node_index_scratch_bytes(n_domains)));
  LWSE_CUDA(e, cudaMemsetAsync(e->node_ix.p, 0, lwse::node_index_scratch_bytes(n_domains), e->stream));
  if (n_nodes)
    LWSE_CUDA(e, cudaMemcpyAsync(e->nodes.p, nodes, (size_t)n_nodes * sizeof(lwse_node_rec),
                                 cudaMemcpyHostToDevice, e->stream));
  e->n_nodes = n_nodes;
  e->n_domains = n_domains;
  e->r_place_current = false;  // (the rows of the last round were computed over the previous node table)
  e->h_nodes.assign(nodes, nodes + n_nodes);
  e->n_usable = 0;
  for (const lwse_node_rec& nd : e->h_nodes) e->n_usable += node_usable(nd, n_domains) ? 1u : 0u;
  e->node_index_stale = true;
  {
    const int rc = build_node_index_locked(e, e->stream, false);
    if (rc != LWSE_OK) return rc;
  }
  if (e->r_loaded && n_nodes) {  // the resident pods' occupancy, counted again for the new table
    LWSE_CUDA(e, e->r_occ.reserve((size_t)n_nodes * 4 + 16));
    LWSE_LAUNCH(e, lwse::launch_occupancy((const lwse_pod_ident*)e->r_pid.p, e->rn_pods, (uint32_t*)e->r_occ.p, n_nodes,
                                          e->sm_count, e->stream));
  }
  LWSE_CUDA(e, cudaStreamSynchronize(e->stream));
  e->place_ns_geometry[0] = e->place_ns_geometry[1] = e->place_ns_geometry[2] = e->place_ns_geometry[3] = 0;
  e->place_geometry[0] = e->place_geometry[1] = e->place_geometry[2] = e->place_geometry[3] = 0;  // re-initialise the scratch
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// LWS sweep
// ---------------------------------------------------------------------------
static int sweep_device_locked(lwse_engine* e, const lwse_lws_tables* t, cudaStream_t s) {
  // the scan bitmaps live in engine-owned scratch; it only grows (a growth is a
  // cudaMalloc, so size it with one warm-up call before capturing a graph)
  LWSE_CUDA(e, e->scan_scratch.reserve(lwse::lws_sweep_scratch_bytes(t->n_pods, t->n_groups)));
  LWSE_LAUNCH(e, lwse::launch_lws_sweep(t, (const lwse_node_rec*)e->nodes.p, e->n_nodes,
                                        e->scan_scratch.p, e->sm_count, s, nullptr));
  return LWSE_OK;
}

LWSE_API int lwse_sweep_lws_device(lwse_engine* e, const lwse_lws_tables* t, void* stream) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  int rc = check_lws_tables(t);
  if (rc != LWSE_OK) return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  return sweep_device_locked(e, t, stream ? (cudaStream_t)stream : e->stream);
}

// lwse_sweep_lws_host with the engine locked and its device current; returns after the results
// are in the caller's tables (stream synchronized — the only synchronize of the call).
// `after_uploads` (optional): called once the table uploads are enqueued and before the sweep is —
// lwse_reconcile_host enqueues its placement branch there, so that the copy engine starts on the
// big tables at once instead of behind the host-side preparation of the round.
static int sweep_host_locked(lwse_engine* e, const lwse_lws_tables* h, const std::function<int()>* after_uploads = nullptr) {
  cudaStream_t s = e->stream;
  const size_t b_lws = (size_t)h->n_lws * sizeof(lwse_lws_rec);
  const size_t b_grp = (size_t)h->n_groups * sizeof(lwse_group_rec);
  const size_t b_pst = (size_t)h->n_pods * sizeof(lwse_pod_state);
  const size_t b_pid = (size_t)h->n_pods * sizeof(lwse_pod_ident);
  const size_t b_lo = (size_t)h->n_lws * sizeof(lwse_lws_out);
  const size_t b_go = (size_t)h->n_groups * sizeof(lwse_group_out);
  LWSE_CUDA(e, e->lws.reserve(b_lws + 16));
  LWSE_CUDA(e, e->groups.reserve(b_grp + 16));
  LWSE_CUDA(e, e->pod_state.reserve(b_pst + 32));
  const void* ident_before = e->pod_ident.p;
  LWSE_CUDA(e, e->pod_ident.reserve(b_pid + 16));
  const bool ident_moved = ident_before != e->pod_ident.p;
  LWSE_CUDA(e, e->scan_scratch.reserve(lwse::lws_sweep_scratch_bytes(h->n_pods, h->n_groups)));
  LWSE_CUDA(e, e->lws_out.reserve(b_lo + 16));
  LWSE_CUDA(e, e->group_out.reserve(b_go + 16));
  const bool want_occ = h->node_occupancy != nullptr && e->n_nodes > 0;
  if (want_occ) {
    LWSE_CUDA(e, e->occupancy.reserve((size_t)e->n_nodes * 4 + 16));
  }
  // the hot byte column first: the identity prefetch below needs only it
  if (b_pst) LWSE_CUDA(e, cudaMemcpyAsync(e->pod_state.p, h->pod_state, b_pst, cudaMemcpyHostToDevice, s));
  lwse_lws_tables d = *h;
  d.lws = (const lwse_lws_rec*)e->lws.p;
  d.groups = (const lwse_group_rec*)e->groups.p;
  d.pod_state = (const lwse_pod_state*)e->pod_state.p;
  d.pod_ident = (const lwse_pod_ident*)e->pod_ident.p;
  d.lws_out = (lwse_lws_out*)e->lws_out.p;
  d.group_out = (lwse_group_out*)e->group_out.p;
  d.node_occupancy = want_occ ? (uint32_t*)e->occupancy.p : nullptr;
  bool counted = false, prefetching = false;
  if (b_pst) {
    // The identity column (16 B / pod, 16 of the 17 input bytes per pod) is only read for pods
    // with a restart / deletion event.  It is left out of the upload
    //  - when the caller says it did not change (LWSE_SWEEP_REUSE_POD_IDENT), or
    //  - when the caller's buffer is pinned, mapped host memory and few pods have an event: a
    //    prefetch kernel on the side stream copies just those rows over PCIe while the other
    //    tables are still being uploaded (a 64-byte read per event pod against 16 B / pod in
    //    bulk).  "Few" is what the PREVIOUS sweep of a table of this size visited (no mid-step
    //    synchronize; the first sweep of a table is optimistic).
    const bool reuse = (h->flags & LWSE_SWEEP_REUSE_POD_IDENT) && e->ident_rows == h->n_pods && !ident_moved;
    const void* mapped = nullptr;
    if (!reuse && !want_occ) {
      cudaPointerAttributes attr;
      if (cudaPointerGetAttributes(&attr, h->pod_ident) == cudaSuccess && attr.type == cudaMemoryTypeHost)
        mapped = attr.devicePointer;
      else
        (void)cudaGetLastError();
    }
    const bool few = e->ident_hint_pods != h->n_pods || (uint64_t)e->ident_hint_events * 64u <= b_pid / 2u;
    if (mapped && few && h->n_groups && !(h->flags & (LWSE_SWEEP_SKIP_POD_SCAN | LWSE_SWEEP_SKIP_GROUP_PASS))) {
      LWSE_CUDA(e, cudaEventRecord(e->ev_fork, s));
      LWSE_CUDA(e, cudaStreamWaitEvent(e->side_stream, e->ev_fork, 0));
      LWSE_LAUNCH(e, lwse::launch_ident_prefetch((const uint8_t*)e->pod_state.p, h->n_pods, (const lwse_pod_ident*)mapped,
                                                 (lwse_pod_ident*)e->pod_ident.p, e->sm_count, e->side_stream));
      LWSE_CUDA(e, cudaEventRecord(e->ev_join, e->side_stream));
      prefetching = true;
      e->ident_rows = ~0ull;  // the device copy holds the event pods' rows only
    } else {
      if (!reuse) LWSE_CUDA(e, cudaMemcpyAsync(e->pod_ident.p, h->pod_ident, b_pid, cudaMemcpyHostToDevice, s));
      e->ident_rows = h->n_pods;
    }
    counted = h->n_groups && !(h->flags & (LWSE_SWEEP_SKIP_POD_SCAN | LWSE_SWEEP_SKIP_GROUP_PASS));
    if (counted) LWSE_CUDA(e, cudaMemsetAsync(e->h_counts_dev.p, 0, 4, s));
  }
  if (b_grp) LWSE_CUDA(e, cudaMemcpyAsync(e->groups.p, h->groups, b_grp, cudaMemcpyHostToDevice, s));
  if (b_lws) LWSE_CUDA(e, cudaMemcpyAsync(e->lws.p, h->lws, b_lws, cudaMemcpyHostToDevice, s));
  if (after_uploads) {
    const int arc = (*after_uploads)();
    if (arc != LWSE_OK) return arc;
  }
  if (prefetching) LWSE_CUDA(e, cudaStreamWaitEvent(s, e->ev_join, 0));
  LWSE_LAUNCH(e, lwse::launch_lws_sweep(&d, (const lwse_node_rec*)e->nodes.p, e->n_nodes, e->scan_scratch.p, e->sm_count,
                                        s, nullptr, counted ? (uint32_t*)e->h_counts_dev.p : nullptr,
                                        /*first_pdl=*/false));

  // group results first: they are complete while the LWS pass still runs
  if (b_go) LWSE_CUDA(e, cudaMemcpyAsync(h->group_out, e->group_out.p, b_go, cudaMemcpyDeviceToHost, s));
  if (b_lo) LWSE_CUDA(e, cudaMemcpyAsync(h->lws_out, e->lws_out.p, b_lo, cudaMemcpyDeviceToHost, s));
  if (want_occ)
    LWSE_CUDA(e, cudaMemcpyAsync(h->node_occupancy, e->occupancy.p, (size_t)e->n_nodes * 4,
                                 cudaMemcpyDeviceToHost, s));
  if (counted) LWSE_CUDA(e, cudaMemcpyAsync(e->h_counts.h, e->h_counts_dev.p, 4, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  if (counted) {
    e->ident_hint_pods = h->n_pods;
    e->ident_hint_events = *static_cast<const uint32_t*>(e->h_counts.h);
  }
  return LWSE_OK;
}

LWSE_API int lwse_sweep_lws_host(lwse_engine* e, const lwse_lws_tables* h) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  int rc = check_lws_tables(h);
  if (rc != LWSE_OK) return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  return sweep_host_locked(e, h);
}

// ---------------------------------------------------------------------------
// Resident tables
// ---------------------------------------------------------------------------
static size_t align256(size_t v) { return (v + 255u) & ~(size_t)255u; }

// (re)allocate the pinned change lists for the resident tables' sizes
static int reserve_change_lists(lwse_engine* e) {
  invalidate_tick_graphs(e);  // called by both resident loads: table pointers and sizes change
  LWSE_CUDA(e, cudaStreamSynchronize(e->pub_stream));  // (a publish kernel may still be copying out of the lists)
  size_t off = 0;
  const size_t sizes[6] = {(size_t)e->rn_lws * 4,       (size_t)e->rn_lws * sizeof(lwse_lws_out),
                           (size_t)e->rn_groups * 4,    (size_t)e->rn_groups * sizeof(lwse_group_out),
                           (size_t)e->rn_reqs * 4,      (size_t)e->rn_reqs * sizeof(lwse_place_out)};
  for (int k = 0; k < 6; k++) {
    e->chg_off[k] = off;
    off += align256(sizes[k] + 16);
  }
  e->chg_bytes = off;
  LWSE_CUDA(e, e->chg.reserve(2 * off));  // two ticks may be in flight: the host reads one slot while the next tick fills the other
  LWSE_CUDA(e, e->chg_dev.reserve(2 * off));  // per tick slot: tick k+1 appends while tick k's lists are published
  LWSE_CUDA(e, e->tickw.reserve(256));
  return LWSE_OK;
}

LWSE_API int lwse_resident_load(lwse_engine* e, const lwse_lws_tables* h) {
  if (!e || !h) return LWSE_ERR_INVALID_ARG;
  if ((h->n_lws && !h->lws) || (h->n_groups && !h->groups) || (h->n_pods && (!h->pod_state || !h->pod_ident)))
    return LWSE_ERR_INVALID_ARG;
  if (h->n_pods > 0xFFFFFFFFull) return LWSE_ERR_UNSUPPORTED;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  {
    const int drc = drain_ticks_locked(e);
    if (drc != LWSE_OK) return drc;
  }
  e->r_swept = false;  // (the output rows are all-ones until the next sweep)
  e->r_groups_swept = false;
  e->r_place_current = false;  // (a new identity column: new occupancy counters)
  cudaStream_t s = e->stream;
  const size_t b_lws = (size_t)h->n_lws * sizeof(lwse_lws_rec), b_grp = (size_t)h->n_groups * sizeof(lwse_group_rec);
  const size_t b_pst = (size_t)h->n_pods * sizeof(lwse_pod_state), b_pid = (size_t)h->n_pods * sizeof(lwse_pod_ident);
  const size_t b_lo = (size_t)h->n_lws * sizeof(lwse_lws_out), b_go = (size_t)h->n_groups * sizeof(lwse_group_out);
  LWSE_CUDA(e, e->r_lws.reserve(b_lws + 16));
  LWSE_CUDA(e, e->r_groups.reserve(b_grp + 16));
  LWSE_CUDA(e, e->r_pst.reserve(b_pst + 32));
  LWSE_CUDA(e, e->r_pid.reserve(b_pid + 16));
  LWSE_CUDA(e, e->r_lws_out.reserve(b_lo + 16));
  LWSE_CUDA(e, e->r_group_out.reserve(b_go + 16));
  LWSE_CUDA(e, e->r_scan.reserve(lwse::lws_sweep_scratch_bytes(h->n_pods, h->n_groups)));
  LWSE_CUDA(e, e->r_counts.reserve(128));  // 64 bytes per tick slot
  LWSE_CUDA(e, e->r_occ.reserve((size_t)e->n_nodes * 4 + 16));
  LWSE_CUDA(e, cudaMemsetAsync(e->r_counts.p, 0, 128, s));
  if (b_lws) LWSE_CUDA(e, cudaMemcpyAsync(e->r_lws.p, h->lws, b_lws, cudaMemcpyHostToDevice, s));
  if (b_grp) LWSE_CUDA(e, cudaMemcpyAsync(e->r_groups.p, h->groups, b_grp, cudaMemcpyHostToDevice, s));
  if (b_pst) LWSE_CUDA(e, cudaMemcpyAsync(e->r_pst.p, h->pod_state, b_pst, cudaMemcpyHostToDevice, s));
  if (b_pid) LWSE_CUDA(e, cudaMemcpyAsync(e->r_pid.p, h->pod_ident, b_pid, cudaMemcpyHostToDevice, s));
  // forget previous results: an all-ones row never equals a real result, so the first sweep reports every row
  if (b_lo) LWSE_CUDA(e, cudaMemsetAsync(e->r_lws_out.p, 0xFF, b_lo, s));
  if (b_go) LWSE_CUDA(e, cudaMemsetAsync(e->r_group_out.p, 0xFF, b_go, s));
  if (e->n_nodes) {  // scheduled pods per node; identity-row patches keep it current from here on
    LWSE_LAUNCH(e, lwse::launch_occupancy((const lwse_pod_ident*)e->r_pid.p, h->n_pods, (uint32_t*)e->r_occ.p, e->n_nodes,
                                          e->sm_count, s));
  }
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  e->rn_lws = h->n_lws;
  e->rn_groups = h->n_groups;
  e->rn_pods = h->n_pods;
  e->r_loaded = true;
  e->r_place_loaded = false;
  e->rn_reqs = 0;
  return reserve_change_lists(e);
}

LWSE_API int lwse_resident_arena(lwse_engine* e, uint64_t min_bytes, void** base_out, uint64_t* bytes_out) {
  if (!e || !base_out) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  const size_t want_arena = min_bytes ? (size_t)min_bytes : ((size_t)8 << 20);
  if (want_arena > e->arena.cap) {  // growing replaces the buffer: nothing may still be reading it
    const int drc = drain_ticks_locked(e);
    if (drc != LWSE_OK) return drc;
    LWSE_CUDA(e, cudaStreamSynchronize(e->stream));
    LWSE_CUDA(e, cudaStreamSynchronize(e->side_stream));
  }
  LWSE_CUDA(e, e->arena.reserve(min_bytes ? (size_t)min_bytes : ((size_t)8 << 20)));
  *base_out = e->arena.h;
  if (bytes_out) *bytes_out = e->arena.cap;
  return LWSE_OK;
}

// table → (device base, rows, bytes per row)
static bool resident_table(lwse_engine* e, uint32_t which, void** base, uint64_t* rows, uint32_t* row_bytes) {
  switch (which) {
    case LWSE_TABLE_LWS: *base = e->r_lws.p; *rows = e->rn_lws; *row_bytes = sizeof(lwse_lws_rec); return true;
    case LWSE_TABLE_GROUPS: *base = e->r_groups.p; *rows = e->rn_groups; *row_bytes = sizeof(lwse_group_rec); return true;
    case LWSE_TABLE_POD_STATE: *base = e->r_pst.p; *rows = e->rn_pods; *row_bytes = sizeof(lwse_pod_state); return true;
    case LWSE_TABLE_POD_IDENT: *base = e->r_pid.p; *rows = e->rn_pods; *row_bytes = sizeof(lwse_pod_ident); return true;
    case LWSE_TABLE_PLACE_REQS:
      if (!e->r_place_loaded) return false;
      *base = e->r_preq.p; *rows = e->rn_reqs; *row_bytes = sizeof(lwse_place_req); return true;
    case LWSE_TABLE_NODES:
      if (e->n_nodes == 0) return false;
      *base = e->nodes.p; *rows = e->n_nodes; *row_bytes = sizeof(lwse_node_rec); return true;
    default: return false;
  }
}

// A segment's rows / values are read by the scatter kernel where the caller wrote them when they
// lie in the arena and are aligned for its vector loads (16-byte row-number reads; 16-byte value
// reads, 4-byte for the byte column); otherwise the call stages a copy.
static bool rows_in_place(const lwse_engine* e, const lwse_patch_seg& g) {
  return e->arena.holds(g.rows, (size_t)g.n * 4) && aligned16(g.rows);
}
static bool values_in_place(const lwse_engine* e, const lwse_patch_seg& g, uint32_t rb) {
  return e->arena.holds(g.values, (size_t)g.n * rb) &&
         (rb == 1 ? (reinterpret_cast<uintptr_t>(g.values) & 3u) == 0 : aligned16(g.values));
}

// What one walk over the segments of a tick (or of lwse_resident_patch, of a what-if) finds: every argument
// check, and what the caller decides from.  The walk writes nothing; commit_segments does, once it passed.
struct SegSummary {
  uint32_t tables = 0;       // bit t: a segment of lwse_table t has rows
  bool any_range = false;    // a LWSE_PATCH_RANGE segment has rows
  bool all_in_place = true;  // no scattered segment needs the staging buffer
  size_t stage_bytes = 0;    // staging the segments outside the arena need
  bool ns_moves = false;     // a request row moves to another namespace
  uint32_t node_rows = 0;    // node rows patched (rows inside the table: the scatter kernel skips the others too)
  bool node_moves = false;   // one of them changes whether its node is usable, or the domain of a usable node
};

static int summarize_segments(lwse_engine* e, const lwse_patch_seg* segs, uint32_t n_segs, SegSummary* out) {
  SegSummary ss;
  if (n_segs && (!segs || n_segs > LWSE_TICK_MAX_SEGS)) return LWSE_ERR_INVALID_ARG;
  for (uint32_t i = 0; i < n_segs; i++) {
    const lwse_patch_seg& g = segs[i];
    void* base;
    uint64_t rows;
    uint32_t rb;
    if (!resident_table(e, g.table, &base, &rows, &rb)) return LWSE_ERR_INVALID_ARG;
    if (g.n == 0) continue;
    const bool range = (g.flags & LWSE_PATCH_RANGE) != 0;
    if (!g.values || (!range && !g.rows)) return LWSE_ERR_INVALID_ARG;
    if (range && (uint64_t)g.first_row + g.n > rows) return LWSE_ERR_BAD_TABLE;
    ss.tables |= 1u << g.table;
    if (range) {
      ss.any_range = true;
    } else {
      if (!rows_in_place(e, g)) ss.stage_bytes += align256((size_t)g.n * 4);
      if (!values_in_place(e, g, rb)) ss.stage_bytes += align256((size_t)g.n * rb);
    }
    if (g.table == LWSE_TABLE_PLACE_REQS) {
      const lwse_place_req* v = static_cast<const lwse_place_req*>(g.values);
      for (uint32_t k = 0; k < g.n && !ss.ns_moves; k++) {
        const uint32_t row = range ? g.first_row + k : g.rows[k];
        ss.ns_moves = row < e->rn_reqs && v[k].ns != e->r_req_ns[row];
      }
    } else if (g.table == LWSE_TABLE_NODES) {
      // (a row patched twice is compared with the mirror both times: some step of old -> v1 -> v2 moves the
      // index exactly when v1 or v2 differs from old in what the index is sorted by)
      const lwse_node_rec* v = static_cast<const lwse_node_rec*>(g.values);
      for (uint32_t k = 0; k < g.n; k++) {
        const uint32_t row = range ? g.first_row + k : g.rows[k];
        if (row >= e->n_nodes) continue;
        ss.node_rows++;
        if (node_patch_moves_index(e->h_nodes[row], v[k], e->n_domains)) ss.node_moves = true;
      }
    }
  }
  ss.all_in_place = ss.stage_bytes == 0;
  *out = ss;
  return LWSE_OK;
}

// The host mirrors follow the segments, once all of them passed their checks: the node table's (and the
// usable-node count; the index is stale when a row moved it) and the request table's namespace column.  A
// request that moves to another namespace breaks the grouping the fast placement kernels rely on, and the
// namespace index of an ungrouped table.
static void commit_segments(lwse_engine* e, const lwse_patch_seg* segs, uint32_t n_segs, const SegSummary& ss) {
  if (ss.node_moves) e->node_index_stale = true;
  for (uint32_t i = 0; i < n_segs; i++) {
    const lwse_patch_seg& g = segs[i];
    const bool nodes = g.table == LWSE_TABLE_NODES && ss.node_rows, reqs = g.table == LWSE_TABLE_PLACE_REQS && ss.ns_moves;
    if (!nodes && !reqs) continue;
    for (uint32_t k = 0; k < g.n; k++) {
      const uint32_t row = (g.flags & LWSE_PATCH_RANGE) ? g.first_row + k : g.rows[k];
      if (nodes && row < e->n_nodes) {
        const lwse_node_rec& now = static_cast<const lwse_node_rec*>(g.values)[k];
        e->n_usable = e->n_usable - (node_usable(e->h_nodes[row], e->n_domains) ? 1u : 0u) + (node_usable(now, e->n_domains) ? 1u : 0u);
        e->h_nodes[row] = now;
      } else if (reqs && row < e->rn_reqs && static_cast<const lwse_place_req*>(g.values)[k].ns != e->r_req_ns[row]) {
        e->r_req_ns[row] = static_cast<const lwse_place_req*>(g.values)[k].ns;
        e->r_place_grouped = false;
        e->r_ns_index_ok = false;
      }
    }
  }
}

// Which resident outputs stop belonging to the resident rows when rows of `tables` are patched and no sweep
// (`swept` false) / no placement round (`placed` false) follows in the same tick.  r_lws_out: the LWS rows (a
// row reused for another object would pass the linked DS tick's uid test with the previous object's results);
// r_group_out: the LWS, group and pod rows; r_pout: the node, request and identity rows a round reads.
static void mark_outputs_stale(lwse_engine* e, uint32_t tables, bool swept, bool placed) {
  constexpr uint32_t kGroupInputs = (1u << LWSE_TABLE_LWS) | (1u << LWSE_TABLE_GROUPS) | (1u << LWSE_TABLE_POD_STATE) | (1u << LWSE_TABLE_POD_IDENT);
  constexpr uint32_t kRoundInputs = (1u << LWSE_TABLE_NODES) | (1u << LWSE_TABLE_PLACE_REQS) | (1u << LWSE_TABLE_POD_IDENT);
  if (!swept && (tables & (1u << LWSE_TABLE_LWS))) e->r_swept = false;
  if (!swept && (tables & kGroupInputs)) e->r_groups_swept = false;
  if (!placed && (tables & kRoundInputs)) e->r_place_current = false;
}

// Room in the staging buffer for the segments that lie outside the arena (rare).  Growing replaces the
// buffer, so nothing may still be reading it.
static int reserve_stage(lwse_engine* e, size_t bytes) {
  if (bytes <= e->stage.cap) return LWSE_OK;
  LWSE_CUDA(e, cudaStreamSynchronize(e->stream));
  LWSE_CUDA(e, cudaStreamSynchronize(e->side_stream));
  LWSE_CUDA(e, e->stage.reserve(bytes));
  return LWSE_OK;
}

// A prepared scatter: where the kernel reads each segment, and the copies that go in front of it.
struct ScatterPlan {
  struct Copy {
    void* dst;
    const void* src;
    size_t bytes;
  };
  lwse::ScatterSegHost sc[LWSE_TICK_MAX_SEGS];
  int n = 0;
  Copy ranges[LWSE_TICK_MAX_SEGS];  // range segments: one DMA copy straight into the table, in segment order
  int n_ranges = 0;
  Copy spans[2];                    // the arena / staging spans the kernel reads from their device mirrors
  int n_spans = 0;
  bool recount = false;             // a range copy rewrote identity rows: the occupancy is counted again
  size_t stage_end = 0;             // the staging buffer is free from here on
};

// Host only: resolves the segments of `tables` (bit t set = lwse_table t; a tick applies the placement request
// patches on the side stream, where the round that reads them runs, and the rest on the engine's stream) to
// device pointers.  Segments outside the arena are copied into the staging buffer from `stage_base` on (the
// caller reserved the room).  Nothing is enqueued.
static int plan_scatter(lwse_engine* e, const lwse_patch_seg* segs, uint32_t n_segs, uint32_t tables, size_t stage_base,
                        size_t dma_min_bytes, ScatterPlan* plan) {
  *plan = ScatterPlan{};
  lwse::ScatterSegHost* sc = plan->sc;
  size_t cursor = stage_base, total = 0;
  for (uint32_t i = 0; i < n_segs; i++) {
    const lwse_patch_seg& g = segs[i];
    if (g.n == 0 || !((tables >> g.table) & 1u)) continue;
    void* base;
    uint64_t rows;
    uint32_t rb;
    if (!resident_table(e, g.table, &base, &rows, &rb)) continue;  // (summarize_segments turns such a segment away)
    if (g.flags & LWSE_PATCH_RANGE) {
      plan->ranges[plan->n_ranges++] = {static_cast<uint8_t*>(base) + (size_t)g.first_row * rb, g.values, (size_t)g.n * rb};
      if (g.table == LWSE_TABLE_POD_IDENT) plan->recount = true;
      continue;
    }
    const void* src[2] = {g.rows, g.values};
    const size_t bytes[2] = {(size_t)g.n * 4, (size_t)g.n * rb};
    const bool in_place[2] = {rows_in_place(e, g), values_in_place(e, g, rb)};
    const void* dev[2];
    for (int c = 0; c < 2; c++) {
      if (in_place[c]) {
        dev[c] = e->arena.dev_of(static_cast<const uint8_t*>(src[c]));
        continue;
      }
      if (cursor + bytes[c] > e->stage.cap) return LWSE_ERR_OOM;
      memcpy(static_cast<uint8_t*>(e->stage.h) + cursor, src[c], bytes[c]);
      dev[c] = static_cast<uint8_t*>(e->stage.d) + cursor;
      cursor += align256(bytes[c]);
    }
    sc[plan->n++] = lwse::ScatterSegHost{base, rows, static_cast<const uint32_t*>(dev[0]), dev[1], g.n, rb, g.table == LWSE_TABLE_POD_IDENT};
    total += bytes[0] + bytes[1];
  }
  plan->stage_end = cursor;
  // Few patch bytes: the scatter kernel reads them in place over PCIe (one round trip, no copy
  // launch).  Many: one DMA copy per pinned buffer of the span this plan uses, then the kernel
  // reads device memory — the copy engine moves large spans several times faster than SM reads of host memory.
  constexpr size_t kDmaBytes = 16384;
  if (plan->n == 0 || total < (dma_min_bytes > kDmaBytes ? dma_min_bytes : kDmaBytes)) return LWSE_OK;
  struct Span { const PinBuf* pin; DevBuf* mirror; uintptr_t lo, hi; } spans[2] = {
      {&e->arena, &e->arena_mirror, UINTPTR_MAX, 0}, {&e->stage, &e->stage_mirror, UINTPTR_MAX, 0}};
  auto touch = [&](const void* dptr, size_t bytes) {
    for (Span& sp : spans) {
      const uintptr_t d0 = reinterpret_cast<uintptr_t>(sp.pin->d), a = reinterpret_cast<uintptr_t>(dptr);
      if (sp.pin->d && a >= d0 && a + bytes <= d0 + sp.pin->cap) {
        sp.lo = a - d0 < sp.lo ? a - d0 : sp.lo;
        sp.hi = a - d0 + bytes > sp.hi ? a - d0 + bytes : sp.hi;
      }
    }
  };
  for (int k = 0; k < plan->n; k++) {
    touch(sc[k].rows, (size_t)sc[k].n * 4);
    touch(sc[k].values, (size_t)sc[k].n * sc[k].row_bytes);
  }
  for (Span& sp : spans) {
    if (sp.hi <= sp.lo) continue;
    if (sp.mirror->cap < sp.pin->cap) {  // (first use, or the pinned buffer grew)
      LWSE_CUDA(e, cudaStreamSynchronize(e->stream));
      LWSE_CUDA(e, cudaStreamSynchronize(e->side_stream));
      LWSE_CUDA(e, cudaStreamSynchronize(e->copy_stream));
      LWSE_CUDA(e, sp.mirror->reserve(sp.pin->cap));
    }
    plan->spans[plan->n_spans++] = {static_cast<uint8_t*>(sp.mirror->p) + sp.lo, static_cast<const uint8_t*>(sp.pin->h) + sp.lo, sp.hi - sp.lo};
    const uintptr_t d0 = reinterpret_cast<uintptr_t>(sp.pin->d), m0 = reinterpret_cast<uintptr_t>(sp.mirror->p);
    for (int k = 0; k < plan->n; k++) {
      uintptr_t a = reinterpret_cast<uintptr_t>(sc[k].rows);
      if (a >= d0 && a < d0 + sp.pin->cap) sc[k].rows = reinterpret_cast<const uint32_t*>(m0 + (a - d0));
      a = reinterpret_cast<uintptr_t>(sc[k].values);
      if (a >= d0 && a < d0 + sp.pin->cap) sc[k].values = reinterpret_cast<const void*>(m0 + (a - d0));
    }
  }
  return LWSE_OK;
}

// The copies of a plan, on `s`: the range segments in segment order, then the mirrored spans.  The scatter
// kernel (launch_scatter_plan, or a tick graph's first node) goes behind all of them.
static int enqueue_scatter_copies(lwse_engine* e, const ScatterPlan& p, cudaStream_t s) {
  for (int k = 0; k < p.n_ranges; k++)
    LWSE_CUDA(e, cudaMemcpyAsync(p.ranges[k].dst, p.ranges[k].src, p.ranges[k].bytes, cudaMemcpyHostToDevice, s));
  for (int k = 0; k < p.n_spans; k++)
    LWSE_CUDA(e, cudaMemcpyAsync(p.spans[k].dst, p.spans[k].src, p.spans[k].bytes, cudaMemcpyHostToDevice, s));
  return LWSE_OK;
}

static int launch_scatter_plan(lwse_engine* e, const ScatterPlan& p, cudaStream_t s) {
  if (p.n) {
    LWSE_LAUNCH(e, lwse::launch_scatter(p.sc, p.n, e->n_nodes ? (uint32_t*)e->r_occ.p : nullptr, e->n_nodes, s, true));
  }
  if (p.recount && e->n_nodes) {
    LWSE_LAUNCH(e, lwse::launch_occupancy((const lwse_pod_ident*)e->r_pid.p, e->rn_pods, (uint32_t*)e->r_occ.p, e->n_nodes,
                                          e->sm_count, s));
  }
  return LWSE_OK;
}

LWSE_API int lwse_resident_patch(lwse_engine* e, lwse_table which, const uint32_t* rows, const void* values,
                                 uint32_t n) {
  if (!e || (n && (!rows || !values))) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  // (node rows only need the node table; the next placement call rebuilds the node index if they ask for it)
  if (which == LWSE_TABLE_NODES ? e->n_nodes == 0 : !e->r_loaded) return LWSE_ERR_NOT_READY;
  if (n == 0) return LWSE_OK;
  DeviceGuard guard(e->device);
  {
    const int drc = drain_ticks_locked(e);
    if (drc != LWSE_OK) return drc;
  }
  lwse_patch_seg seg{};
  seg.table = (uint32_t)which;
  seg.n = n;
  seg.rows = rows;
  seg.values = values;
  SegSummary ss;
  if (const int crc = summarize_segments(e, &seg, 1, &ss); crc != LWSE_OK) return crc;
  // the round of the last placement call may still read the node rows (and it reads them on another stream)
  if (which == LWSE_TABLE_NODES && e->place_pending) LWSE_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_place, 0));
  commit_segments(e, &seg, 1, ss);
  mark_outputs_stale(e, ss.tables, false, false);
  ScatterPlan plan;
  int rc = reserve_stage(e, ss.stage_bytes);
  if (rc == LWSE_OK) rc = plan_scatter(e, &seg, 1, ss.tables, 0, 0, &plan);
  if (rc == LWSE_OK) rc = enqueue_scatter_copies(e, plan, e->stream);
  if (rc == LWSE_OK) rc = launch_scatter_plan(e, plan, e->stream);
  if (rc != LWSE_OK) {
    if (which == LWSE_TABLE_NODES) e->node_index_stale = true;  // (see tick_submit_locked)
    return rc;
  }
  // the caller's buffers (and the staging copy) are free again once the scatter ran
  LWSE_CUDA(e, cudaStreamSynchronize(e->stream));
  return LWSE_OK;
}

LWSE_API int lwse_resident_outputs(lwse_engine* e, lwse_lws_out* lws_out, lwse_group_out* group_out) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  cudaStream_t s = e->stream;
  if (lws_out && e->rn_lws)
    LWSE_CUDA(e, cudaMemcpyAsync(lws_out, e->r_lws_out.p, (size_t)e->rn_lws * sizeof(lwse_lws_out), cudaMemcpyDeviceToHost, s));
  if (group_out && e->rn_groups)
    LWSE_CUDA(e, cudaMemcpyAsync(group_out, e->r_group_out.p, (size_t)e->rn_groups * sizeof(lwse_group_out),
                                 cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Placement
// ---------------------------------------------------------------------------
constexpr uint32_t kFormGeneral = 0, kFormGrouped = 1, kFormScan = 2;

// The namespace-parallel form (request table grouped by namespace): condense kernel + one CTA per
// namespace.  `first_pdl`: nothing on the stream right before writes the request table.  `index` other
// than kNsIndexNone: the resident request table, not grouped — the indexed form.
static int place_grouped_locked(lwse_engine* e, const lwse_place_req* d_reqs, uint32_t n_reqs, const uint32_t* d_occupancy,
                                uint32_t n_parts, uint64_t part_stride_bytes, uint32_t n_namespaces, lwse_place_out* d_out,
                                bool scan, uint32_t* rounds_out, uint32_t* scans_out, cudaStream_t s, bool first_pdl,
                                const lwse::PlaceNsChanges* changes = nullptr, const lwse::PlaceNsExchange* xch = nullptr,
                                lwse::PlaceNsIndex index = lwse::kNsIndexNone) {
  const size_t scratch = lwse::place_ns_scratch_bytes(e->n_nodes, e->n_domains, n_reqs, n_namespaces);
  const void* before = e->place_ns_scratch.p;
  LWSE_CUDA(e, e->place_ns_scratch.reserve(scratch));
  const uint32_t geometry[4] = {n_reqs, n_namespaces, e->n_nodes, e->n_domains};
  const bool fresh = before != e->place_ns_scratch.p || memcmp(geometry, e->place_ns_geometry, sizeof(geometry)) != 0;
  memcpy(e->place_ns_geometry, geometry, sizeof(geometry));
  cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
  const bool eager = cudaStreamIsCapturing(s, &capturing) == cudaSuccess && capturing == cudaStreamCaptureStatusNone;
  if (fresh && eager) invalidate_tick_graphs(e);  // (their kernel nodes hold the old scratch pointers)
  if (eager && e->place_pending) LWSE_CUDA(e, cudaStreamWaitEvent(s, e->ev_place, 0));
  bool built = false;
  {
    const int rc = build_node_index_locked(e, s, false, &built);
    if (rc != LWSE_OK) return rc;
  }
  const uint32_t* counters = nullptr;
  LWSE_LAUNCH(e, lwse::launch_place_ns((const lwse_node_rec*)e->nodes.p, (const uint32_t*)e->dom_first.p,
                                       (const uint32_t*)e->node_order.p, e->n_nodes, e->n_domains, d_reqs, n_reqs,
                                       d_occupancy, n_parts, part_stride_bytes, n_namespaces, d_out, e->place_ns_scratch.p,
                                       scratch, fresh, e->place_ns_calls++, scan, e->sm_count, s, &counters,
                                       (first_pdl || built) && !fresh, changes, xch, index));
  e->r_ns_index_ok = index != lwse::kNsIndexNone;  // (a grouped call writes its own ns_first over the index's)
  e->place_rounds_ptr = counters;
  e->place_scans_ptr = counters + 3;
  if (eager && !changes) {  // (a tick — `changes` — returns only after the host has seen the round complete)
    LWSE_CUDA(e, cudaEventRecord(e->ev_place, s));
    e->place_pending = true;
  }
  if (rounds_out) {
    uint32_t* const h_rounds = static_cast<uint32_t*>(e->h_rounds.h);
    LWSE_CUDA(e, cudaMemcpyAsync(h_rounds + 4, counters, 16, cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaStreamSynchronize(s));
    *rounds_out = h_rounds[4];
    if (scans_out) *scans_out = h_rounds[7];
  }
  return LWSE_OK;
}

static int place_locked(lwse_engine* e, const lwse_place_req* d_reqs, uint32_t n_reqs,
                        const uint32_t* d_occupancy, uint32_t n_namespaces, lwse_place_out* d_out,
                        uint32_t* rounds_out, cudaStream_t s, uint32_t n_parts, uint32_t reqs_per_part,
                        uint64_t part_stride_bytes, bool after_push = false, uint32_t form = kFormGeneral,
                        bool first_pdl = false, const lwse::PlaceNsChanges* changes = nullptr, bool* diffed = nullptr,
                        lwse::PlaceNsIndex index = lwse::kNsIndexNone) {
  if ((n_reqs && (!d_reqs || !d_out)) || n_namespaces == 0) return LWSE_ERR_INVALID_ARG;
  if (e->n_nodes == 0 || e->n_domains == 0) return LWSE_ERR_NOT_READY;
  if (diffed) *diffed = false;
  if (form != kFormGeneral && n_parts <= 1 && lwse::place_ns_supported(e->n_nodes, e->n_domains)) {
    if (diffed) *diffed = changes != nullptr;
    return place_grouped_locked(e, d_reqs, n_reqs, d_occupancy, 1, 0, n_namespaces, d_out, form == kFormScan, rounds_out, nullptr,
                                s, first_pdl, changes, nullptr, index);
  }
  const size_t scratch = lwse::place_scratch_bytes(e->n_nodes, e->n_domains, n_reqs, n_namespaces);
  const void* before = e->place_scratch.p;
  LWSE_CUDA(e, e->place_scratch.reserve(scratch));
  // the two scratch halves are laid out for one geometry; any change re-initialises them
  const uint32_t geometry[4] = {n_reqs, n_namespaces, e->n_nodes, e->n_domains};
  const bool fresh = before != e->place_scratch.p || memcmp(geometry, e->place_geometry, sizeof(geometry)) != 0;
  uint32_t* const h_rounds = static_cast<uint32_t*>(e->h_rounds.h);
  if (fresh) h_rounds[2] = 0xFFFFFFFFu;  // no history for this geometry
  memcpy(e->place_geometry, geometry, sizeof(geometry));
  // placement calls of one engine share the scratch (a call resets the half the next one uses):
  // whatever streams they run on, each orders behind the previous one
  cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
  const bool eager = cudaStreamIsCapturing(s, &capturing) == cudaSuccess && capturing == cudaStreamCaptureStatusNone;
  if (eager && e->place_pending) LWSE_CUDA(e, cudaStreamWaitEvent(s, e->ev_place, 0));
  {
    const int rc = build_node_index_locked(e, s, false);
    if (rc != LWSE_OK) return rc;
  }
  LWSE_LAUNCH(e, lwse::launch_place((const lwse_node_rec*)e->nodes.p, (const uint32_t*)e->dom_first.p,
                                    (const uint32_t*)e->node_order.p, (const uint32_t*)e->node_pos.p, e->n_nodes,
                                    e->n_domains, d_reqs,
                                    n_reqs, d_occupancy, n_namespaces, d_out, e->place_scratch.p,
                                    scratch, rounds_out ? h_rounds : nullptr, e->sm_count, s,
                                    e->place_calls++, fresh, n_parts, reqs_per_part, part_stride_bytes,
                                    h_rounds + 2, &e->place_counters, &e->place_unpinned, after_push));
  e->place_rounds_ptr = e->place_counters + 3;
  e->place_scans_ptr = nullptr;
  if (rounds_out) *rounds_out = h_rounds[0];
  if (eager) {
    LWSE_CUDA(e, cudaEventRecord(e->ev_place, s));
    e->place_pending = true;
  }
  // history for the next call's cluster-or-grid decision (only consulted beyond 1024 requests):
  // the round's unpinned-request count, copied on a third stream so that nothing waits for it
  if (n_reqs > 1024u && e->place_unpinned && eager) {
    LWSE_CUDA(e, cudaStreamWaitEvent(e->hist_stream, e->ev_place, 0));
    LWSE_CUDA(e, cudaMemcpyAsync(h_rounds + 2, e->place_unpinned, 4, cudaMemcpyDeviceToHost, e->hist_stream));
  }
  return LWSE_OK;
}

// ns non-decreasing over the table?  (host tables: a 4-byte read per 32-byte row)
static bool grouped_by_namespace(const lwse_place_req* reqs, uint32_t n) {
  for (uint32_t i = 1; i < n; i++)
    if (reqs[i].ns < reqs[i - 1].ns) return false;
  return true;
}

static uint32_t form_of_flags(uint32_t sweep_flags) {
  if (!(sweep_flags & LWSE_SWEEP_PLACE_GROUPED)) return kFormGeneral;
  return (sweep_flags & LWSE_SWEEP_PLACE_SCAN) ? kFormScan : kFormGrouped;
}

static int place_common(lwse_engine* e, const lwse_place_req* d_reqs, uint32_t n_reqs,
                        const uint32_t* d_occupancy, uint32_t n_namespaces, lwse_place_out* d_out,
                        uint32_t* rounds_out, void* stream, uint32_t n_parts, uint32_t reqs_per_part,
                        uint64_t part_stride_bytes) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  return place_locked(e, d_reqs, n_reqs, d_occupancy, n_namespaces, d_out, rounds_out,
                      stream ? (cudaStream_t)stream : e->stream, n_parts, reqs_per_part, part_stride_bytes);
}

// One reconcile tick on device tables: the placement round reads only inputs (requests, occupancy,
// node table), never the sweep's outputs, so it is enqueued on the engine's side stream and runs
// concurrently with the three sweep kernels; `stream` continues when both are done.
LWSE_API int lwse_reconcile_device(lwse_engine* e, const lwse_lws_tables* t, const lwse_place_req* d_reqs,
                                   uint32_t n_reqs, const uint32_t* d_occupancy, uint32_t n_namespaces,
                                   lwse_place_out* d_place_out, void* stream) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  int rc = check_lws_tables(t);
  if (rc != LWSE_OK) return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  cudaStream_t s = stream ? (cudaStream_t)stream : e->stream;
  if (n_reqs == 0) return sweep_device_locked(e, t, s);
  LWSE_CUDA(e, cudaEventRecord(e->ev_fork, s));
  LWSE_CUDA(e, cudaStreamWaitEvent(e->side_stream, e->ev_fork, 0));
  rc = place_locked(e, d_reqs, n_reqs, d_occupancy, n_namespaces, d_place_out, nullptr, e->side_stream, 1, n_reqs, 0, false,
                    form_of_flags(t->flags), /*first_pdl=*/false);
  if (rc == LWSE_OK) rc = sweep_device_locked(e, t, s);
  // join even after a failure, so that the side stream never runs ahead of `stream`
  cudaError_t je = cudaEventRecord(e->ev_join, e->side_stream);
  if (je == cudaSuccess) je = cudaStreamWaitEvent(s, e->ev_join, 0);
  if (rc != LWSE_OK) return rc;
  if (je != cudaSuccess) return fail_cuda(e, je);
  return LWSE_OK;
}

LWSE_API int lwse_place_device(lwse_engine* e, const lwse_place_req* d_reqs, uint32_t n_reqs,
                               const uint32_t* d_occupancy, uint32_t n_namespaces,
                               lwse_place_out* d_out, uint32_t* rounds_out, void* stream) {
  return place_common(e, d_reqs, n_reqs, d_occupancy, n_namespaces, d_out, rounds_out, stream, 1, n_reqs, 0);
}

LWSE_API int lwse_place_grouped_device(lwse_engine* e, const lwse_place_req* d_reqs, uint32_t n_reqs,
                                       const uint32_t* d_occupancy, uint32_t n_namespaces, lwse_place_out* d_out,
                                       uint32_t flags, uint32_t* rounds_out, uint32_t* pair_scans_out, void* stream) {
  if (!e || (n_reqs && (!d_reqs || !d_out)) || n_namespaces == 0) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (e->n_nodes == 0 || e->n_domains == 0) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  cudaStream_t s = stream ? (cudaStream_t)stream : e->stream;
  if (!lwse::place_ns_supported(e->n_nodes, e->n_domains))  // too many domains for one CTA's shared memory
    return place_locked(e, d_reqs, n_reqs, d_occupancy, n_namespaces, d_out, rounds_out, s, 1, n_reqs, 0);
  return place_grouped_locked(e, d_reqs, n_reqs, d_occupancy, 1, 0, n_namespaces, d_out, (flags & LWSE_SWEEP_PLACE_SCAN) != 0,
                              rounds_out, pair_scans_out, s, /*first_pdl=*/false);
}

LWSE_API int lwse_place_gathered_device(lwse_engine* e, const void* d_parts, uint32_t n_parts,
                                        uint64_t part_stride_bytes, uint64_t reqs_offset_bytes,
                                        uint32_t reqs_per_part, uint32_t n_namespaces,
                                        lwse_place_out* d_out, uint32_t* rounds_out, void* stream) {
  if (!d_parts || n_parts == 0 || (part_stride_bytes & 15u) || (reqs_offset_bytes & 15u) ||
      (uint64_t)n_parts * reqs_per_part > 0xFFFFFFull)
    return LWSE_ERR_INVALID_ARG;
  const uint8_t* base = static_cast<const uint8_t*>(d_parts);
  return place_common(e, reinterpret_cast<const lwse_place_req*>(base + reqs_offset_bytes), n_parts * reqs_per_part,
                      reinterpret_cast<const uint32_t*>(base), n_namespaces, d_out, rounds_out, stream, n_parts,
                      reqs_per_part, part_stride_bytes);
}

// ---------------------------------------------------------------------------
// Peer exchange (multi-GPU placement step)
// ---------------------------------------------------------------------------
LWSE_API int lwse_exchange_create(lwse_engine* e, uint32_t reqs_per_part, uint32_t world, uint32_t rank,
                                  void* handle_out) {
  if (!e || !handle_out || world == 0 || world > LWSE_MAX_RANKS || rank >= world) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (e->n_nodes == 0 || e->n_domains == 0) return LWSE_ERR_NOT_READY;
  if (e->xch_world) return LWSE_ERR_UNSUPPORTED;  // one exchange per engine
  DeviceGuard guard(e->device);
  const uint64_t reqs_off = ((uint64_t)e->n_nodes * 4u + 15u) / 16u * 16u;
  const uint64_t stride = reqs_off + (uint64_t)reqs_per_part * sizeof(lwse_place_req);
  const uint64_t half = ((uint64_t)world * stride + 255u) / 256u * 256u;
  const uint64_t flags_off = 3u * half;  // three buffers: step s uses buffer s % 3 (lwse_exchange_kernels.cu)
  const uint64_t total = flags_off + (uint64_t)world * 8u + 64u;
  LWSE_CUDA(e, e->xch.reserve(total));
  LWSE_CUDA(e, cudaMemset(e->xch.p, 0, total));
  LWSE_CUDA(e, e->xch_peers_dev.reserve(sizeof(void*) * LWSE_MAX_RANKS));
  cudaIpcMemHandle_t h;
  LWSE_CUDA(e, cudaIpcGetMemHandle(&h, e->xch.p));
  static_assert(sizeof(h) == LWSE_IPC_HANDLE_BYTES, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle_out, &h, sizeof(h));
  e->xch_world = world;
  e->xch_rank = rank;
  e->xch_reqs_per_part = reqs_per_part;
  e->xch_stride = stride;
  e->xch_reqs_off = reqs_off;
  e->xch_half = half;
  e->xch_flags_off = flags_off;
  e->xch_step = 0;
  e->xch_connected = false;
  return LWSE_OK;
}

LWSE_API int lwse_exchange_connect(lwse_engine* e, const void* handles) {
  if (!e || !handles) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->xch_world || e->xch_connected) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  cudaError_t err = cudaSuccess;
  for (uint32_t p = 0; err == cudaSuccess && p < e->xch_world; p++) {
    if (p == e->xch_rank) {
      e->xch_peer.p[p] = e->xch.p;
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, static_cast<const uint8_t*>(handles) + (size_t)p * LWSE_IPC_HANDLE_BYTES, sizeof(h));
    err = e->xch_peer.open(p, h);
  }
  if (err == cudaSuccess)
    err = cudaMemcpy(e->xch_peers_dev.p, e->xch_peer.p, sizeof(void*) * e->xch_world, cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    e->xch_peer.close();  // a retry starts from no mappings
    return fail_cuda(e, err);
  }
  e->xch_connected = true;
  return LWSE_OK;
}

LWSE_API uint64_t lwse_exchange_part_bytes(const lwse_engine* e) { return e ? e->xch_stride : 0; }

// One reconcile tick of a multi-GPU shard: as lwse_reconcile_device, with the placement round
// solved over every rank's part — this rank's part is pushed to all peers first.
LWSE_API int lwse_reconcile_exchanged_device(lwse_engine* e, const lwse_lws_tables* t, const void* d_local_part,
                                             uint32_t n_namespaces, lwse_place_out* d_place_out, void* stream) {
  if (!e || !d_local_part || !aligned16(d_local_part)) return LWSE_ERR_INVALID_ARG;
  int rc = t ? check_lws_tables(t) : LWSE_OK;
  if (rc != LWSE_OK) return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->xch_connected) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  cudaStream_t s = stream ? (cudaStream_t)stream : e->stream;
  LWSE_CUDA(e, cudaEventRecord(e->ev_fork, s));
  LWSE_CUDA(e, cudaStreamWaitEvent(e->side_stream, e->ev_fork, 0));
  const uint64_t step = ++e->xch_step;
  rc = count_launch(e, lwse::launch_exchange_push(d_local_part, (uint8_t* const*)e->xch_peers_dev.p, e->xch.p,
                                                 e->xch_stride, e->xch_stride, e->xch_half, e->xch_flags_off, step,
                                                 step, e->xch_world, e->xch_rank, e->side_stream, false));
  if (rc == LWSE_OK) {
    const uint8_t* half = static_cast<const uint8_t*>(e->xch.p) + (step % 3ull) * e->xch_half;
    rc = place_locked(e, reinterpret_cast<const lwse_place_req*>(half + e->xch_reqs_off),
                      e->xch_world * e->xch_reqs_per_part, reinterpret_cast<const uint32_t*>(half), n_namespaces,
                      d_place_out, nullptr, e->side_stream, e->xch_world, e->xch_reqs_per_part, e->xch_stride,
                      /*after_push=*/true);
  }
  if (rc == LWSE_OK && t) rc = sweep_device_locked(e, t, s);
  cudaError_t je = cudaEventRecord(e->ev_join, e->side_stream);
  if (je == cudaSuccess) je = cudaStreamWaitEvent(s, e->ev_join, 0);
  if (rc != LWSE_OK) return rc;
  if (je != cudaSuccess) return fail_cuda(e, je);
  return LWSE_OK;
}

// The placement branch of a tick whose requests are LOCAL and whose occupancy is shared: push this
// rank's occupancy counters to every peer, then solve the local requests against the sum of all
// ranks' counters.  Enqueued on `ps`.  lagged: read the previous step's snapshot (see the kernel file).
static int shared_occupancy_place_locked(lwse_engine* e, const lwse_place_req* d_reqs, uint32_t n_reqs,
                                         const uint32_t* d_local_occ, uint32_t n_namespaces, lwse_place_out* d_out,
                                         uint32_t form, bool lagged, cudaStream_t ps,
                                         const lwse::PlaceNsChanges* changes = nullptr,
                                         lwse::PlaceNsIndex index = lwse::kNsIndexNone) {
  // While a tick graph is being captured the step is not a parameter: the push kernel takes it from
  // the device counter every push advances (and the condense kernel the blocks to sum from the same
  // counter), so that the replayed nodes follow the step; the replay itself advances e->xch_step.
  cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
  const bool eager = cudaStreamIsCapturing(ps, &capturing) == cudaSuccess && capturing == cudaStreamCaptureStatusNone;
  const uint64_t step = eager ? ++e->xch_step : 0ull;
  const uint64_t read_step = (lagged && step > 1) ? step - 1 : step;
  LWSE_LAUNCH(e, lwse::launch_exchange_push(d_local_occ, (uint8_t* const*)e->xch_peers_dev.p, e->xch.p,
                                            e->xch_reqs_off,  // the occupancy block of a part: n_nodes counters, 16-byte padded
                                            e->xch_stride, e->xch_half, e->xch_flags_off, step, read_step, e->xch_world,
                                            e->xch_rank, ps, lagged));
  if (n_reqs == 0) return LWSE_OK;
  const lwse::PlaceNsExchange xch{reinterpret_cast<const unsigned long long*>(static_cast<const uint8_t*>(e->xch.p) + e->xch_flags_off +
                                                                              (uint64_t)e->xch_world * 8u + 16u),
                                  e->xch_half, lagged};
  if (form != kFormGeneral && lwse::place_ns_supported(e->n_nodes, e->n_domains))
    return place_grouped_locked(e, d_reqs, n_reqs, static_cast<const uint32_t*>(e->xch.p), e->xch_world, e->xch_stride, n_namespaces,
                                d_out, form == kFormScan, nullptr, nullptr, ps, /*first_pdl=*/true, changes, &xch,
                                index);  // behind the push kernel
  return LWSE_ERR_UNSUPPORTED;  // the shared-occupancy form needs a request table grouped by namespace
}

LWSE_API int lwse_reconcile_shared_device(lwse_engine* e, const lwse_lws_tables* t, const lwse_place_req* d_reqs,
                                          uint32_t n_reqs, const uint32_t* d_local_occupancy, uint32_t n_namespaces,
                                          lwse_place_out* d_place_out, uint32_t flags, void* stream) {
  if (!e || !d_local_occupancy || !aligned16(d_local_occupancy) || (n_reqs && (!d_reqs || !d_place_out)) || n_namespaces == 0)
    return LWSE_ERR_INVALID_ARG;
  int rc = t ? check_lws_tables(t) : LWSE_OK;
  if (rc != LWSE_OK) return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->xch_connected) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  cudaStream_t s = stream ? (cudaStream_t)stream : e->stream;
  LWSE_CUDA(e, cudaEventRecord(e->ev_fork, s));
  LWSE_CUDA(e, cudaStreamWaitEvent(e->side_stream, e->ev_fork, 0));
  rc = shared_occupancy_place_locked(e, d_reqs, n_reqs, d_local_occupancy, n_namespaces, d_place_out,
                                     (flags & LWSE_SWEEP_PLACE_SCAN) ? kFormScan : kFormGrouped,
                                     (flags & LWSE_EXCHANGE_LAGGED) != 0, e->side_stream);
  if (rc == LWSE_OK && t) rc = sweep_device_locked(e, t, s);
  cudaError_t je = cudaEventRecord(e->ev_join, e->side_stream);
  if (je == cudaSuccess) je = cudaStreamWaitEvent(s, e->ev_join, 0);
  if (rc != LWSE_OK) return rc;
  if (je != cudaSuccess) return fail_cuda(e, je);
  return LWSE_OK;
}

// 0 = every wait so far saw all peers; 1 = a wait timed out (a peer is gone).  Synchronizes.
LWSE_API int lwse_exchange_status(lwse_engine* e, uint32_t* error_out) {
  if (!e || !error_out) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->xch_world) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, cudaDeviceSynchronize());
  LWSE_CUDA(e, cudaMemcpy(error_out, static_cast<const uint8_t*>(e->xch.p) + e->xch_flags_off + (uint64_t)e->xch_world * 8u + 4u,
                          4, cudaMemcpyDeviceToHost));
  return LWSE_OK;
}

// Measurement aid (not part of lwse.h): with LWSE_WHATIF_TIMING=1, the device time of the last what-if on its
// stream, from behind the snapshot event to the end of the diff kernel (the copies back to the host excluded).
extern "C" __attribute__((visibility("default"))) int lwse_debug_whatif_device_us(lwse_engine* e, float* us) {
  if (!e || !us) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->wf_timed) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  float ms = 0.f;
  LWSE_CUDA(e, cudaEventElapsedTime(&ms, e->ev_wf_t0, e->ev_wf_t1));
  *us = ms * 1000.f;
  return LWSE_OK;
}

// Test aid (not part of lwse.h): copies the first n_rows rows of a resident input table (LWSE_TABLE_LWS, _GROUPS,
// _POD_STATE, _POD_IDENT, or a DS table including LWSE_TABLE_DS_LINKS) to host memory, after the device is idle.
// Tests read the tables back to check that a call left them as they were.
extern "C" __attribute__((visibility("default"))) int lwse_debug_resident_read(lwse_engine* e, uint32_t table, void* out,
                                                                               uint32_t n_rows) {
  if (!e || (n_rows && !out)) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  void* base = nullptr;
  uint32_t rows = 0, rb = 0;
  switch (table) {
    case LWSE_TABLE_LWS: base = e->r_lws.p; rows = e->rn_lws; rb = sizeof(lwse_lws_rec); break;
    case LWSE_TABLE_GROUPS: base = e->r_groups.p; rows = e->rn_groups; rb = sizeof(lwse_group_rec); break;
    case LWSE_TABLE_POD_STATE: base = e->r_pst.p; rows = (uint32_t)e->rn_pods; rb = 1; break;
    case LWSE_TABLE_POD_IDENT: base = e->r_pid.p; rows = (uint32_t)e->rn_pods; rb = sizeof(lwse_pod_ident); break;
    default:
      if (!e->rd_loaded || !ds_resident_table(e, table, &base, &rows, &rb)) return LWSE_ERR_INVALID_ARG;
  }
  if (table <= LWSE_TABLE_POD_IDENT && !e->r_loaded) return LWSE_ERR_NOT_READY;
  if (n_rows > rows) return LWSE_ERR_INVALID_ARG;
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, cudaDeviceSynchronize());
  if (n_rows) LWSE_CUDA(e, cudaMemcpy(out, base, (size_t)n_rows * rb, cudaMemcpyDeviceToHost));
  return LWSE_OK;
}

// Test aid (not part of lwse.h): the CUDA objects all engines of the process hold (allocations, streams, events,
// graph executables, peer mappings).  Tests check that a closed engine gave back all of its own.
extern "C" __attribute__((visibility("default"))) int64_t lwse_debug_cuda_objects(void) { return g_cuda_objects.load(); }

// Tuning aid (not part of lwse.h): phase timestamps of the most recent placement kernel.
extern "C" __attribute__((visibility("default"))) int lwse_debug_place_trace(lwse_engine* e, uint64_t* out16) {
  if (!e || !out16 || !e->place_scratch.p || e->place_calls == 0) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  cudaDeviceSynchronize();
  // the half used by the last call: layout [holder | counters …]; holder size is unknown here, so the
  // launcher recorded the counters pointer
  if (!e->place_counters) return LWSE_ERR_NOT_READY;
  uint32_t raw[32];
  if (cudaMemcpy(raw, e->place_counters + 16, sizeof(raw), cudaMemcpyDeviceToHost) != cudaSuccess)
    return LWSE_ERR_CUDA;
  for (int k = 0; k < 16; k++) out16[k] = (uint64_t)raw[2 * k] | ((uint64_t)raw[2 * k + 1] << 32);
  return LWSE_OK;
}

LWSE_API int lwse_place_host(lwse_engine* e, const lwse_place_req* reqs, uint32_t n_reqs,
                             const uint32_t* occupancy, uint32_t n_namespaces, lwse_place_out* out,
                             uint32_t* rounds_out) {
  if (!e || (n_reqs && (!reqs || !out)) || n_namespaces == 0) return LWSE_ERR_INVALID_ARG;
  // one lock for staging, launch and download: concurrent callers (Go reconcile workers) share
  // the staging buffers
  std::lock_guard<std::mutex> lock(e->mu);
  if (e->n_nodes == 0 || e->n_domains == 0) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  cudaStream_t s = e->stream;
  LWSE_CUDA(e, e->place_reqs.reserve((size_t)n_reqs * sizeof(lwse_place_req) + 16));
  LWSE_CUDA(e, e->place_out.reserve((size_t)n_reqs * sizeof(lwse_place_out) + 16));
  LWSE_CUDA(e, e->place_occ.reserve((size_t)e->n_nodes * 4 + 16));
  if (n_reqs)
    LWSE_CUDA(e, cudaMemcpyAsync(e->place_reqs.p, reqs, (size_t)n_reqs * sizeof(lwse_place_req), cudaMemcpyHostToDevice, s));
  if (occupancy)
    LWSE_CUDA(e, cudaMemcpyAsync(e->place_occ.p, occupancy, (size_t)e->n_nodes * 4, cudaMemcpyHostToDevice, s));
  else
    LWSE_CUDA(e, cudaMemsetAsync(e->place_occ.p, 0, (size_t)e->n_nodes * 4, s));
  // a table grouped by namespace (the encoder emits it that way) takes the namespace-parallel kernels
  const uint32_t form = n_reqs && grouped_by_namespace(reqs, n_reqs) ? kFormGrouped : kFormGeneral;
  const int rc = place_locked(e, (const lwse_place_req*)e->place_reqs.p, n_reqs, (const uint32_t*)e->place_occ.p, n_namespaces,
                              (lwse_place_out*)e->place_out.p, rounds_out, s, 1, n_reqs, 0, false, form);
  if (rc != LWSE_OK) return rc;
  if (n_reqs)
    LWSE_CUDA(e, cudaMemcpyAsync(out, e->place_out.p, (size_t)n_reqs * sizeof(lwse_place_out), cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  return LWSE_OK;
}

// One reconcile tick from host tables: lwse_sweep_lws_host and lwse_place_host in one call.  The
// placement round (its inputs are 70 KB) is uploaded, solved and read back on the side stream
// while the tables of the sweep are still crossing PCIe; one synchronize at the end.
LWSE_API int lwse_reconcile_host(lwse_engine* e, const lwse_lws_tables* h, const lwse_place_req* reqs,
                                 uint32_t n_reqs, const uint32_t* occupancy, uint32_t n_namespaces,
                                 lwse_place_out* place_out) {
  if (!e || (n_reqs && (!reqs || !place_out || n_namespaces == 0))) return LWSE_ERR_INVALID_ARG;
  int rc = check_lws_tables(h);
  if (rc != LWSE_OK) return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  if (n_reqs && (e->n_nodes == 0 || e->n_domains == 0)) return LWSE_ERR_NOT_READY;
  // LWSE_SWEEP_PLACE_GROUPED: the caller promises a request table grouped by namespace (the encoder
  // emits it that way) — no host pass over the table; the condense kernel counts order violations
  // and a broken promise comes back as LWSE_ERR_BAD_TABLE.
  const bool promised = n_reqs && (h->flags & LWSE_SWEEP_PLACE_GROUPED) && lwse::place_ns_supported(e->n_nodes, e->n_domains);
  bool check_order = false;
  const std::function<int()> place_branch = [&]() -> int {
    if (!n_reqs) return LWSE_OK;
    cudaStream_t ps = e->side_stream;
    LWSE_CUDA(e, e->place_reqs.reserve((size_t)n_reqs * sizeof(lwse_place_req) + 16));
    LWSE_CUDA(e, e->place_out.reserve((size_t)n_reqs * sizeof(lwse_place_out) + 16));
    LWSE_CUDA(e, e->place_occ.reserve((size_t)e->n_nodes * 4 + 16));
    // (the side stream only ever runs work enqueued under this lock and joined before it is released)
    LWSE_CUDA(e, cudaMemcpyAsync(e->place_reqs.p, reqs, (size_t)n_reqs * sizeof(lwse_place_req), cudaMemcpyHostToDevice, ps));
    if (occupancy)
      LWSE_CUDA(e, cudaMemcpyAsync(e->place_occ.p, occupancy, (size_t)e->n_nodes * 4, cudaMemcpyHostToDevice, ps));
    else
      LWSE_CUDA(e, cudaMemsetAsync(e->place_occ.p, 0, (size_t)e->n_nodes * 4, ps));
    const bool grouped = promised || grouped_by_namespace(reqs, n_reqs);
    const uint32_t form = grouped ? ((h->flags & LWSE_SWEEP_PLACE_SCAN) ? kFormScan : kFormGrouped) : kFormGeneral;
    const int prc = place_locked(e, (const lwse_place_req*)e->place_reqs.p, n_reqs, (const uint32_t*)e->place_occ.p, n_namespaces,
                                 (lwse_place_out*)e->place_out.p, nullptr, ps, 1, n_reqs, 0, false, form);
    if (prc != LWSE_OK) return prc;
    if (promised && e->place_scans_ptr != nullptr) {  // (the namespace kernels ran: their counter block)
      LWSE_CUDA(e, cudaMemcpyAsync(static_cast<uint32_t*>(e->h_rounds.h) + 8, e->place_rounds_ptr + 2, 4, cudaMemcpyDeviceToHost, ps));
      check_order = true;
    }
    LWSE_CUDA(e, cudaMemcpyAsync(place_out, e->place_out.p, (size_t)n_reqs * sizeof(lwse_place_out), cudaMemcpyDeviceToHost, ps));
    return LWSE_OK;
  };
  const int rc_sweep = sweep_host_locked(e, h, &place_branch);
  if (n_reqs) {
    const cudaError_t pe = cudaStreamSynchronize(e->side_stream);
    if (rc_sweep == LWSE_OK && pe != cudaSuccess) return fail_cuda(e, pe);
    if (rc_sweep == LWSE_OK && check_order && static_cast<const uint32_t*>(e->h_rounds.h)[8] != 0u) return LWSE_ERR_BAD_TABLE;
  }
  return rc_sweep;
}

// ---------------------------------------------------------------------------
// The resident tick
// ---------------------------------------------------------------------------
LWSE_API int lwse_resident_place_load(lwse_engine* e, const lwse_place_req* reqs, uint32_t n_reqs,
                                      uint32_t n_namespaces) {
  if (!e || (n_reqs && !reqs) || n_namespaces == 0 || !aligned16(reqs)) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded || e->n_nodes == 0 || e->n_domains == 0) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  {
    const int drc = drain_ticks_locked(e);
    if (drc != LWSE_OK) return drc;
    LWSE_CUDA(e, cudaStreamSynchronize(e->side_stream));
  }
  cudaStream_t s = e->stream;
  const size_t b_req = (size_t)n_reqs * sizeof(lwse_place_req), b_out = (size_t)n_reqs * sizeof(lwse_place_out);
  LWSE_CUDA(e, e->r_preq.reserve(b_req + 16));
  LWSE_CUDA(e, e->r_pout.reserve(b_out + 16));
  LWSE_CUDA(e, e->r_pout_prev.reserve(b_out + 16));
  if (b_req) LWSE_CUDA(e, cudaMemcpyAsync(e->r_preq.p, reqs, b_req, cudaMemcpyHostToDevice, s));
  if (b_out) LWSE_CUDA(e, cudaMemsetAsync(e->r_pout_prev.p, 0xFF, b_out, s));  // the first tick reports every row
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  e->rn_reqs = n_reqs;
  e->rn_namespaces = n_namespaces;
  e->r_place_loaded = true;
  e->r_place_current = false;  // (no round over these rows yet)
  e->r_place_grouped = grouped_by_namespace(reqs, n_reqs);
  e->r_ns_index_ok = false;  // an ungrouped table: the first tick builds the namespace index
  e->r_req_ns.resize(n_reqs);
  for (uint32_t i = 0; i < n_reqs; i++) e->r_req_ns[i] = reqs[i].ns;
  return reserve_change_lists(e);
}

static inline void cpu_relax() {
#if defined(__x86_64__) || defined(__i386__)
  __builtin_ia32_pause();
#endif
}

// Spin until the device has raised *w to `seq` (mapped host memory).  While waiting, look at the
// stream now and then: a faulted kernel never raises the word.  false = error or 10 s without news.
static bool wait_word(volatile uint32_t* w, uint32_t seq, cudaStream_t s, cudaError_t* err) {
  *err = cudaSuccess;
  const auto t0 = std::chrono::steady_clock::now();
  for (uint64_t it = 1;; it++) {
    if (*w == seq) {
      std::atomic_thread_fence(std::memory_order_acquire);
      return true;
    }
    cpu_relax();
    if ((it & 0x3FFFu) == 0) {
      const cudaError_t q = cudaStreamQuery(s);
      if (q != cudaSuccess && q != cudaErrorNotReady) {
        *err = q;
        return false;
      }
      if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > 10.0) return *w == seq;
    }
  }
}

struct TickCounts {
  uint32_t n_lws = 0, n_groups = 0, n_place = 0, rounds = 0;
};

static inline uint8_t* d_desc_of(lwse_engine* e, uint32_t slot) {
  return static_cast<uint8_t*>(e->tdesc_dev.p) + slot * lwse::kScatterDescBytes;
}

// The patches of a tick go where their readers run: the placement request table is read only by the round
// on the side stream, everything else by the sweep on the engine's stream.
constexpr uint32_t kSideTables = 1u << LWSE_TABLE_PLACE_REQS;

// Every decision of one tick, made by plan_tick before anything is enqueued.  The enqueue functions, the
// graph key, lwse_tick_info and the slot's bookkeeping all read it and nothing else.
struct TickPlan {
  uint32_t slot = 0;         // t_submitted & 1: which pinned lists, words and counters the tick uses
  bool in_flight = false;    // the previous tick has not been waited for yet
  bool do_sweep = false, do_place = false;
  bool round_asked = false;  // LWSE_TICK_PLACE on a loaded request table: r_pout is current afterwards (trivially so for an empty table)
  uint32_t sweep_flags = 0;  // LWSE_SWEEP_GANG
  // The round's form.  A request table grouped by namespace — and not ungrouped by this tick's patches — runs
  // the namespace kernels as they are; any other table runs them through the namespace index, rebuilt when the
  // namespace column changed since the last build.  The general form only where the namespace form cannot run.
  bool ns_form = false, scan_form = false, indexed = false;
  lwse::PlaceNsIndex ns_index = lwse::kNsIndexNone;
  bool shared_occ = false, lagged = false;  // LWSE_TICK_SHARED_OCCUPANCY (and its LWSE_EXCHANGE_LAGGED)
  bool has_patches = false, has_ident = false, has_side = false;
  bool wrote_main = false;   // a table is patched on the engine's stream
  uint32_t node_rows = 0;
  bool node_rebuild = false;  // the round rebuilds the node index (a tick without a round leaves a stale index to the next one)
  // A round forks behind the engine's stream when it reads what the main scatter writes — identity-row patches
  // move occupancy counts, node-row patches change the nodes — or when an earlier tick without a round patched
  // tables there that no round has been ordered behind yet.
  bool prior_unforked = false, fork_behind_main = false;
  // LWSE_TICK_GRAPH: 1 = replay when the previous tick is still in flight — the pipelined use, where the host's
  // enqueue time is what limits the rate; a lone tick is faster kernel by kernel, because its round starts
  // while the copy engine still moves the pod patches; 2 = always; 0 = never.  Only ticks whose patches all lie
  // in the arena, and whose round takes the namespace form, are replayed.
  bool graph_ok = false;
};

static TickPlan plan_tick(const lwse_engine* e, const SegSummary& ss, uint32_t flags) {
  TickPlan p;
  p.slot = (uint32_t)(e->t_submitted & 1u);
  p.in_flight = e->t_submitted != e->t_waited;
  p.round_asked = (flags & LWSE_TICK_PLACE) && e->r_place_loaded;
  p.do_place = p.round_asked && e->rn_reqs > 0;
  p.do_sweep = !(flags & LWSE_TICK_NO_SWEEP) && (e->rn_lws || e->rn_groups);
  p.sweep_flags = flags & LWSE_SWEEP_GANG;
  p.ns_form = p.do_place && lwse::place_ns_supported(e->n_nodes, e->n_domains);
  p.scan_form = (flags & LWSE_SWEEP_PLACE_SCAN) != 0;
  p.indexed = p.ns_form && !(e->r_place_grouped && !ss.ns_moves);
  p.ns_index = !p.indexed                             ? lwse::kNsIndexNone
               : (ss.ns_moves || !e->r_ns_index_ok) ? lwse::kNsIndexBuild
                                                      : lwse::kNsIndexReuse;
  p.shared_occ = (flags & LWSE_TICK_SHARED_OCCUPANCY) != 0;
  p.lagged = p.shared_occ && (flags & LWSE_EXCHANGE_LAGGED);
  p.has_patches = ss.tables != 0;
  p.has_ident = (ss.tables & (1u << LWSE_TABLE_POD_IDENT)) != 0;
  p.has_side = (ss.tables & kSideTables) != 0;
  p.wrote_main = (ss.tables & ~kSideTables) != 0;
  p.node_rows = ss.node_rows;
  p.node_rebuild = p.do_place && (e->node_index_stale || ss.node_moves);
  p.prior_unforked = p.do_place && e->main_unforked;
  p.fork_behind_main = p.has_ident || p.node_rows > 0 || p.prior_unforked;
  p.graph_ok = (e->use_graph >= 2 || (e->use_graph == 1 && p.in_flight)) && ss.all_in_place && !ss.any_range &&
               (!p.shared_occ || (p.do_place && e->xch_connected)) && (p.do_sweep || p.do_place) &&
               !(p.has_side && !p.do_place) && (!p.do_place || p.ns_form);
  return p;
}

// One graph per shape of the tick and slot: every decision that changes what a replayable tick enqueues has
// its bit here.  (has_ident, has_side and the forks do not: a graph's one scatter takes every table, and its
// round always forks behind it.)
static uint32_t graph_key(const TickPlan& p) {
  enum { kPatches, kSweep, kPlace, kGang, kScan, kSlot, kSharedOcc, kLagged, kIndexed, kIndexBuild, kNodeRows, kNodeRebuild };
  auto bit = [](bool on, int at) { return (on ? 1u : 0u) << at; };
  return bit(p.has_patches, kPatches) | bit(p.do_sweep, kSweep) | bit(p.do_place, kPlace) | bit(p.sweep_flags != 0, kGang) |
         bit(p.scan_form, kScan) | bit(p.slot != 0, kSlot) | bit(p.shared_occ, kSharedOcc) | bit(p.lagged, kLagged) |
         bit(p.indexed, kIndexed) | bit(p.ns_index == lwse::kNsIndexBuild, kIndexBuild) | bit(p.node_rows > 0, kNodeRows) |
         bit(p.node_rebuild, kNodeRebuild);
}

static lwse_tick_info tick_info(const TickPlan& p, bool graph) {
  lwse_tick_info ti{};
  ti.place_form = !p.do_place   ? LWSE_TICK_FORM_NONE
                  : !p.ns_form  ? LWSE_TICK_FORM_GENERAL
                  : p.scan_form ? LWSE_TICK_FORM_SCAN
                                : LWSE_TICK_FORM_NAMESPACE;
  ti.indexed = p.indexed ? 1u : 0u;
  ti.index_built = p.ns_index == lwse::kNsIndexBuild ? 1u : 0u;
  ti.graph = graph ? 1u : 0u;
  return ti;
}

// The bookkeeping that closes a submitted tick.
static void close_submit(lwse_engine* e, const TickPlan& p, uint32_t seq, bool graph) {
  lwse_engine::TickSlot& ts = e->tslot[p.slot];
  ts.seq = seq;
  ts.do_sweep = p.do_sweep;
  ts.do_place = p.do_place;
  ts.published = p.do_sweep || p.do_place;
  ts.wrote = p.has_patches;
  e->t_submitted++;
  if (p.do_sweep) {
    e->r_swept = e->r_groups_swept = true;
    e->r_sweep_flags = p.sweep_flags;
  }
  if (p.round_asked) e->r_place_current = true;
  e->main_unforked = !p.do_place && (e->main_unforked || p.wrote_main);
  e->last_tick_info = tick_info(p, graph);
  if (p.indexed) e->r_ns_index_ok = true;  // (also after a replay, which enqueues no call that would say so)
}

// One tick slot's buffers: its words in pinned memory, its pinned change lists (both as the device sees them),
// the device-memory lists the kernels append to, and their counters.
struct SlotBufs {
  uint32_t* words;
  uint8_t *chg_pinned, *chg_dev;
  uint32_t* counts;
};
static SlotBufs slot_bufs(const lwse_engine* e, uint32_t slot) {
  return {static_cast<uint32_t*>(e->tickw.d) + slot * 16u, static_cast<uint8_t*>(e->chg.d) + slot * e->chg_bytes,
          static_cast<uint8_t*>(e->chg_dev.p) + slot * e->chg_bytes, static_cast<uint32_t*>(e->r_counts.p) + slot * 16u};
}

// `first_mode`: how the sweep's first kernel is launched (see launch_lws_sweep): 2 behind this tick's scatter
// kernel alone (programmatic: it waits at its top), 1 eager with nothing to wait for, 0 behind an event or as a
// graph's first node (ordinary).
static int enqueue_sweep(lwse_engine* e, const TickPlan& p, int first_mode) {
  const SlotBufs b = slot_bufs(e, p.slot);
  lwse_lws_tables d{};
  d.lws = (const lwse_lws_rec*)e->r_lws.p;
  d.n_lws = e->rn_lws;
  d.groups = (const lwse_group_rec*)e->r_groups.p;
  d.n_groups = e->rn_groups;
  d.pod_state = (const lwse_pod_state*)e->r_pst.p;
  d.pod_ident = (const lwse_pod_ident*)e->r_pid.p;
  d.n_pods = e->rn_pods;
  d.lws_out = (lwse_lws_out*)e->r_lws_out.p;
  d.group_out = (lwse_group_out*)e->r_group_out.p;
  d.flags = p.sweep_flags;
  lwse::SweepChangeLists cl;
  cl.lws_rows = reinterpret_cast<uint32_t*>(b.chg_dev + e->chg_off[0]);
  cl.lws_out = reinterpret_cast<lwse_lws_out*>(b.chg_dev + e->chg_off[1]);
  cl.lws_capacity = e->rn_lws;
  cl.group_rows = reinterpret_cast<uint32_t*>(b.chg_dev + e->chg_off[2]);
  cl.group_out = reinterpret_cast<lwse_group_out*>(b.chg_dev + e->chg_off[3]);
  cl.group_capacity = e->rn_groups;
  cl.counts = b.counts;
  return count_launch(e, lwse::launch_lws_sweep(&d, (const lwse_node_rec*)e->nodes.p, e->n_nodes, e->r_scan.p, e->sm_count,
                                                e->stream, &cl, nullptr, first_mode));
}

// How the round's first kernels are launched.  Eagerly the first one follows a kernel on the side stream; in a
// graph capture it follows an event (an ordinary launch), and `mid_event` is recorded between the condense and
// the namespace kernel.
struct PlaceLaunch {
  bool first_pdl;
  void* mid_event;
};

static int enqueue_place(lwse_engine* e, const TickPlan& p, const PlaceLaunch& how, TickPlaceResult* res) {
  const SlotBufs b = slot_bufs(e, p.slot);
  cudaStream_t ps = e->side_stream;
  const uint32_t form = !p.ns_form ? kFormGeneral : p.scan_form ? kFormScan : kFormGrouped;
  // the namespace kernels append the changed rows themselves; the general form gets a diff kernel
  const lwse::PlaceNsChanges changes{(lwse_place_out*)e->r_pout_prev.p, reinterpret_cast<uint32_t*>(b.chg_dev + e->chg_off[4]),
                                     reinterpret_cast<lwse_place_out*>(b.chg_dev + e->chg_off[5]), b.counts + 4, e->rn_reqs,
                                     (int)p.slot, how.mid_event};
  bool diffed = false;
  int rc;
  if (p.shared_occ) {  // multi-rank: this rank's counters go to the peers, the round sees the sum
    if (!e->xch_connected) return LWSE_ERR_NOT_READY;
    rc = shared_occupancy_place_locked(e, (const lwse_place_req*)e->r_preq.p, e->rn_reqs, (const uint32_t*)e->r_occ.p,
                                       e->rn_namespaces, (lwse_place_out*)e->r_pout.p, form, p.lagged, ps, &changes, p.ns_index);
    diffed = rc == LWSE_OK;
  } else {
    rc = place_locked(e, (const lwse_place_req*)e->r_preq.p, e->rn_reqs, (const uint32_t*)e->r_occ.p, e->rn_namespaces,
                      (lwse_place_out*)e->r_pout.p, nullptr, ps, 1, e->rn_reqs, 0, false, form, how.first_pdl, &changes, &diffed,
                      p.ns_index);
  }
  if (rc != LWSE_OK) return rc;
  if (!diffed) {
    LWSE_LAUNCH(e, lwse::launch_place_diff((const lwse_place_out*)e->r_pout.p, changes.prev, e->rn_reqs, changes.rows,
                                           changes.outs, changes.capacity, changes.count, ps));
  }
  *res = TickPlaceResult{diffed, e->place_rounds_ptr};
  return LWSE_OK;
}

// The tick's last step, on the publish stream: behind everything the tick enqueued on the engine's
// stream (both branches joined there), so the NEXT tick's kernels do not wait for the copy of this
// tick's changed rows to the host.  ONE kernel copies all change lists out (0 LWS rows, 1 group rows,
// 2 placement rows); lists, counters and the round's counter block are per slot.
static int enqueue_publish(lwse_engine* e, const TickPlan& p, uint32_t seq, const TickPlaceResult& placed) {
  const SlotBufs b = slot_bufs(e, p.slot);
  const uint32_t capacity[3] = {e->rn_lws, e->rn_groups, e->rn_reqs};
  const uint32_t out_bytes[3] = {sizeof(lwse_lws_out), sizeof(lwse_group_out), sizeof(lwse_place_out)};
  lwse::PublishListHost pl[3] = {};
  for (int k = 0; k < 3; k++)
    if (k == 2 ? p.do_place : p.do_sweep)
      pl[k] = {reinterpret_cast<uint32_t*>(b.chg_dev + e->chg_off[2 * k]), b.chg_dev + e->chg_off[2 * k + 1],
               reinterpret_cast<uint32_t*>(b.chg_pinned + e->chg_off[2 * k]), b.chg_pinned + e->chg_off[2 * k + 1],
               b.counts + (k == 2 ? 4 : k), capacity[k], out_bytes[k]};
  LWSE_CUDA(e, cudaEventRecord(e->ev_done, e->stream));
  LWSE_CUDA(e, cudaStreamWaitEvent(e->pub_stream, e->ev_done, 0));
  const uint32_t* rounds = p.do_place ? placed.rounds_ptr : nullptr;
  LWSE_LAUNCH(e, lwse::launch_publish(pl, rounds, b.words, 4, seq, b.counts + 2, e->last_changed[0] + e->last_changed[1],
                                      e->pub_stream, p.do_place && placed.place_ns ? const_cast<uint32_t*>(rounds) : nullptr, 8u,
                                      /*pdl=*/false));
  LWSE_CUDA(e, cudaEventRecord(e->ev_pub, e->pub_stream));
  return LWSE_OK;
}

// The graph of plan `p`, captured from the same enqueue functions on capturing streams:
//   scatter (from the slot's descriptor block) -> condense -> { fused -> LWS pass  ||  namespace kernel }.
// Returns an error only when the streams could not be drained; a capture that fails leaves tg.exec null and
// the key eager for good (the streams are usable again after EndCapture).
static int capture_tick_graph(lwse_engine* e, const TickPlan& p, lwse_engine::TickGraph& tg) {
  cudaStream_t s = e->stream, ps = e->side_stream;
  cudaError_t ce = cudaStreamSynchronize(s);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(ps);
  if (ce != cudaSuccess) return fail_cuda(e, ce);
  const uint64_t launches_before = e->launches;
  int crc = LWSE_OK;
  TickPlaceResult placed;
  ce = cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed);
  if (ce == cudaSuccess) {
    auto cap = [&](cudaError_t x) { if (crc == LWSE_OK && x != cudaSuccess) { ce = x; crc = LWSE_ERR_CUDA; } };
    if (p.has_patches) {  // the graph's first node: an ordinary launch
      const int launched = lwse::launch_scatter_desc(d_desc_of(e, p.slot), e->sm_count, s, /*pdl=*/false);
      if (launched < 0) cap((cudaError_t)-launched); else e->launches += (uint64_t)launched;
    }
    if (p.do_place) {  // the round forks behind the scatter (it reads the request rows and the occupancy counters)
      cap(cudaEventRecord(e->ev_fork, s));
      cap(cudaStreamWaitEvent(ps, e->ev_fork, 0));
      // The fused sweep kernel fills every SM (3 CTAs of 256 x 77 registers) the moment it starts
      // and the namespace kernel's CTAs (512 x 53 registers) then wait for CTAs to retire: hold
      // the sweep back until the (short) condense kernel is done, so that both reach the SMs together.
      if (crc == LWSE_OK) crc = enqueue_place(e, p, PlaceLaunch{false, p.do_sweep ? (void*)e->ev_mid : nullptr}, &placed);
      if (p.do_sweep && placed.place_ns) cap(cudaStreamWaitEvent(s, e->ev_mid, 0));
    }
    if (crc == LWSE_OK && p.do_sweep) crc = enqueue_sweep(e, p, (p.has_patches && !placed.place_ns) ? 2 : 0);
    if (p.do_place) {
      cap(cudaEventRecord(e->ev_join, ps));
      cap(cudaStreamWaitEvent(s, e->ev_join, 0));
    }
    cudaGraph_t graph = nullptr;
    const cudaError_t ee = cudaStreamEndCapture(s, &graph);
    if (ee != cudaSuccess || graph == nullptr) cap(ee != cudaSuccess ? ee : cudaErrorUnknown);
    if (crc == LWSE_OK) cap(tg.exec.ensure(graph));
    if (graph) cudaGraphDestroy(graph);
  } else {
    crc = LWSE_ERR_CUDA;
  }
  tg.kernels = (uint32_t)(e->launches - launches_before);
  e->launches = launches_before;
  if (crc != LWSE_OK || !tg.exec) {
    (void)cudaGetLastError();
    tg.exec.reset();
    tg.failed = true;
    e->node_index_stale = e->node_index_stale || p.node_rebuild;  // (the eager run builds it)
  } else {
    tg.place = placed;
  }
  return LWSE_OK;
}

// Enqueueing a tick kernel by kernel costs ~10 runtime calls of microseconds each (launches with
// attributes and 200-400 bytes of parameters): more host time than the GPU needs for the tick.
// A tick whose plan allows it (graph_ok) is therefore replayed as ONE graph per key, from the second tick
// of that key on: the first runs eagerly, so that every buffer settles.
// What changes from tick to tick travels outside the graph, on the copy stream, so that the
// copies of tick k+1 overlap the kernels of tick k: the patch bytes (arena span -> mirror, one scatter for
// every table behind one copy) and the scatter's segment descriptors (a 512-byte block, pinned slot ->
// device).  The publish kernel follows on the publish stream, launched with the tick's sequence number.
// *done: the tick was enqueued; otherwise the caller enqueues it eagerly.
static int replay_tick(lwse_engine* e, const TickPlan& p, const lwse_patch_seg* segs, uint32_t n_segs, uint32_t seq, bool* done) {
  *done = false;
  lwse_engine::TickGraph& tg = e->tick_graphs[graph_key(p)];
  if (tg.seen++ == 0 || tg.failed) return LWSE_OK;
  ScatterPlan gp;
  if (const int rc = plan_scatter(e, segs, n_segs, 0xFFFFFFFFu, 0, 0, &gp); rc != LWSE_OK) return rc;
  const size_t desc_bytes = lwse::kScatterDescBytes;
  if (e->tdesc.reserve(2 * desc_bytes) != cudaSuccess || e->tdesc_dev.reserve(2 * desc_bytes) != cudaSuccess) {
    (void)cudaGetLastError();
    return LWSE_OK;
  }
  uint8_t* h_desc = static_cast<uint8_t*>(e->tdesc.h) + p.slot * desc_bytes;
  if (p.has_patches && !lwse::write_scatter_desc(h_desc, gp.sc, gp.n, e->n_nodes ? (uint32_t*)e->r_occ.p : nullptr, e->n_nodes))
    return LWSE_OK;
  if (!tg.exec) {
    if (const int rc = capture_tick_graph(e, p, tg); rc != LWSE_OK) return rc;
    if (!tg.exec) return LWSE_OK;
  }
  if (p.has_patches) {
    if (const int rc = enqueue_scatter_copies(e, gp, e->copy_stream); rc != LWSE_OK) return rc;
    LWSE_CUDA(e, cudaMemcpyAsync(d_desc_of(e, p.slot), h_desc, desc_bytes, cudaMemcpyHostToDevice, e->copy_stream));
    LWSE_CUDA(e, cudaEventRecord(e->ev_dma, e->copy_stream));
    LWSE_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_dma, 0));
  }
  LWSE_CUDA(e, cudaGraphLaunch(tg.exec, e->stream));
  e->launches += tg.kernels;
  if (p.node_rebuild) e->node_index_stale = false;  // (the graph's round built it)
  e->graph_ticks++;
  if (p.shared_occ) e->xch_step++;  // (the replayed push kernel advanced the device counter by one)
  if (p.do_place) e->place_rounds_ptr = tg.place.rounds_ptr;
  if (const int rc = enqueue_publish(e, p, seq, tg.place); rc != LWSE_OK) return rc;
  close_submit(e, p, seq, true);
  *done = true;
  return LWSE_OK;
}

// The eager enqueue order.  Every call costs microseconds of host time and the copy of the pod patches
// heads the critical path, so that copy is enqueued first; the round's launches follow on the side
// stream while the copy engine works — it starts behind its own few request rows (read in place over PCIe:
// no copy-engine launch) and is mostly done when the sweep needs the SMs — then the main scatter and the
// sweep behind the copy.  A round that forks behind the main scatter needs that scatter enqueued before it,
// so the scatter keeps its place in front then.
static int enqueue_tick_eager(lwse_engine* e, const TickPlan& p, const lwse_patch_seg* segs, uint32_t n_segs, uint32_t seq) {
  cudaStream_t s = e->stream, ps = e->side_stream;
  const bool scatter_last = !p.fork_behind_main;
  ScatterPlan main_plan, side_plan;
  int rc = plan_scatter(e, segs, n_segs, ~kSideTables, 0, 0, &main_plan);
  if (rc == LWSE_OK) rc = enqueue_scatter_copies(e, main_plan, s);
  if (rc == LWSE_OK && !scatter_last) rc = launch_scatter_plan(e, main_plan, s);
  if (rc != LWSE_OK) return rc;
  if (p.fork_behind_main && (p.wrote_main || p.prior_unforked) && (p.has_side || p.do_place)) {
    LWSE_CUDA(e, cudaEventRecord(e->ev_fork, s));
    LWSE_CUDA(e, cudaStreamWaitEvent(ps, e->ev_fork, 0));
  }
  if (p.has_side) {
    rc = plan_scatter(e, segs, n_segs, kSideTables, main_plan.stage_end, /*dma_min_bytes=*/65536, &side_plan);
    if (rc == LWSE_OK) rc = enqueue_scatter_copies(e, side_plan, ps);
    if (rc == LWSE_OK) rc = launch_scatter_plan(e, side_plan, ps);
  }
  const PlaceLaunch how{/*first_pdl=*/true, /*mid_event=*/nullptr};
  TickPlaceResult placed;
  if (rc == LWSE_OK && p.do_place && p.wrote_main) rc = enqueue_place(e, p, how, &placed);
  if (rc == LWSE_OK && scatter_last) rc = launch_scatter_plan(e, main_plan, s);
  if (rc == LWSE_OK && p.do_sweep) rc = enqueue_sweep(e, p, p.wrote_main ? 2 : 1);
  if (rc == LWSE_OK && p.do_place && !p.wrote_main) rc = enqueue_place(e, p, how, &placed);
  if (rc != LWSE_OK) return rc;
  if (p.do_place || p.has_side) {
    LWSE_CUDA(e, cudaEventRecord(e->ev_join, ps));
    LWSE_CUDA(e, cudaStreamWaitEvent(s, e->ev_join, 0));
  }
  if (p.do_sweep || p.do_place) {
    rc = enqueue_publish(e, p, seq, placed);
    if (rc != LWSE_OK) return rc;
  }
  close_submit(e, p, seq, false);
  return LWSE_OK;
}

// Decide one tick, then enqueue it (nothing waits): slot = t_submitted & 1.  At most two ticks are in flight.
// Argument errors come back before anything changes.
static int submit_tick(lwse_engine* e, const lwse_patch_seg* segs, uint32_t n_segs, uint32_t flags) {
  if (e->t_submitted - e->t_waited >= 2) return LWSE_ERR_NOT_READY;  // wait for the oldest tick first
  SegSummary ss;
  if (const int rc = summarize_segments(e, segs, n_segs, &ss); rc != LWSE_OK) return rc;
  const TickPlan p = plan_tick(e, ss, flags);
  mark_outputs_stale(e, ss.tables, p.do_sweep, p.round_asked);
  commit_segments(e, segs, n_segs, ss);
  e->last_node_info = lwse_node_info{p.node_rows, p.node_rebuild ? 1u : 0u, e->n_usable, 0u};
  // sequence numbers count the ticks that end in a publish kernel (the device counts the same ones)
  uint32_t seq = 0;
  if (p.do_sweep || p.do_place) {
    seq = ++e->tick_seq;
    if (seq == 0) seq = ++e->tick_seq;
  }
  if (const int rc = reserve_stage(e, ss.stage_bytes); rc != LWSE_OK) return rc;
  if (p.in_flight) {
    // a tick is still running.  Its DMA may still read the staging buffer: segments outside the arena
    // wait for it.
    if (!ss.all_in_place) {
      LWSE_CUDA(e, cudaStreamSynchronize(e->stream));
      LWSE_CUDA(e, cudaStreamSynchronize(e->side_stream));
    }
    // the general placement kernel keeps its counters in two alternating scratch halves (a call resets
    // the half the next one uses): its round may not start before the previous tick's publish kernel
    // has read them.  (The namespace kernels count in the tick slot's own block.)
    if (p.do_place && !p.ns_form) LWSE_CUDA(e, cudaStreamWaitEvent(e->side_stream, e->ev_pub, 0));
  }
  if (p.graph_ok) {
    bool done = false;
    const int rc = replay_tick(e, p, segs, n_segs, seq, &done);
    if (rc != LWSE_OK || done) return rc;
  }
  return enqueue_tick_eager(e, p, segs, n_segs, seq);
}

static int tick_submit_locked(lwse_engine* e, const lwse_patch_seg* segs, uint32_t n_segs, uint32_t flags) {
  const int rc = submit_tick(e, segs, n_segs, flags);
  if (rc != LWSE_OK) e->r_place_current = false;  // (its patches may or may not have been applied)
  if (rc != LWSE_OK && segs) {
    // A tick that fails once its node rows are in the mirror (a CUDA error, no staging memory) may or may
    // not have patched them on the device: the next round rebuilds the index from the device rows.
    for (uint32_t i = 0; i < n_segs && i < LWSE_TICK_MAX_SEGS; i++)
      if (segs[i].table == LWSE_TABLE_NODES && segs[i].n) e->node_index_stale = true;
  }
  return rc;
}

// The oldest tick in flight: spin on its sequence word (the tick's only wait), report its counts.
static int tick_wait_locked(lwse_engine* e, TickCounts* out, uint32_t* slot_out) {
  if (e->t_submitted == e->t_waited) return LWSE_ERR_NOT_READY;
  const uint32_t slot = (uint32_t)(e->t_waited & 1u);
  const lwse_engine::TickSlot ts = e->tslot[slot];
  cudaStream_t s = e->stream;
  volatile uint32_t* hw = static_cast<volatile uint32_t*>(e->tickw.h) + slot * 16u;
  cudaError_t werr = cudaSuccess;
  bool ok = true;
  if (ts.published) {
    ok = wait_word(hw + 4, ts.seq, s, &werr);
  } else if (ts.wrote) {
    werr = cudaStreamSynchronize(s);
    ok = werr == cudaSuccess;
  }
  e->t_waited++;
  if (!ok) {
    const cudaError_t a = cudaStreamSynchronize(s), b = cudaStreamSynchronize(e->side_stream);
    e->t_waited = e->t_submitted;  // whatever else was in flight died with it
    return fail_cuda(e, werr != cudaSuccess ? werr : a != cudaSuccess ? a : b != cudaSuccess ? b : cudaErrorUnknown);
  }
  if (ts.do_place && e->t_submitted == e->t_waited) e->place_pending = false;  // the publish kernel ran behind the join: the round is complete
  out->n_lws = ts.do_sweep ? hw[0] : 0u;
  out->n_groups = ts.do_sweep ? hw[1] : 0u;
  out->n_place = ts.do_place ? hw[2] : 0u;
  out->rounds = ts.do_place ? hw[3] : 0u;
  e->last_changed[0] = out->n_lws + out->n_groups;
  e->last_changed[1] = out->n_place;
  if (slot_out) *slot_out = slot;
  return LWSE_OK;
}

static void fill_tick_outputs(const lwse_engine* e, uint32_t slot, const TickCounts& c, lwse_tick* t) {
  const uint8_t* base = static_cast<const uint8_t*>(e->chg.h) + slot * e->chg_bytes;
  t->lws_rows = reinterpret_cast<const uint32_t*>(base + e->chg_off[0]);
  t->lws_out = reinterpret_cast<const lwse_lws_out*>(base + e->chg_off[1]);
  t->group_rows = reinterpret_cast<const uint32_t*>(base + e->chg_off[2]);
  t->group_out = reinterpret_cast<const lwse_group_out*>(base + e->chg_off[3]);
  t->place_rows = reinterpret_cast<const uint32_t*>(base + e->chg_off[4]);
  t->place_out = reinterpret_cast<const lwse_place_out*>(base + e->chg_off[5]);
  t->n_lws = c.n_lws;
  t->n_groups = c.n_groups;
  t->n_place = c.n_place;
  t->place_rounds = c.rounds;
}

// Every tick in flight is waited for (its results are dropped): the synchronous entry points call this first.
static int drain_ticks_locked(lwse_engine* e) {
  while (e->t_submitted != e->t_waited) {
    TickCounts c;
    const int rc = tick_wait_locked(e, &c, nullptr);
    if (rc != LWSE_OK) return rc;
  }
  return LWSE_OK;
}

LWSE_API int lwse_resident_tick(lwse_engine* e, lwse_tick* t) {
  if (!e || !t || (t->n_segs && !t->segs)) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  int rc = drain_ticks_locked(e);
  if (rc != LWSE_OK) return rc;
  rc = tick_submit_locked(e, t->segs, t->n_segs, t->flags);
  if (rc != LWSE_OK) return rc;
  TickCounts c;
  uint32_t slot = 0;
  rc = tick_wait_locked(e, &c, &slot);
  if (rc != LWSE_OK) return rc;
  fill_tick_outputs(e, slot, c, t);
  return LWSE_OK;
}

LWSE_API int lwse_resident_tick_submit(lwse_engine* e, const lwse_tick* t) {
  if (!e || !t || (t->n_segs && !t->segs)) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  return tick_submit_locked(e, t->segs, t->n_segs, t->flags);
}

LWSE_API int lwse_resident_tick_wait(lwse_engine* e, lwse_tick* t) {
  if (!e || !t) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  TickCounts c;
  uint32_t slot = 0;
  const int rc = tick_wait_locked(e, &c, &slot);
  if (rc != LWSE_OK) return rc;
  fill_tick_outputs(e, slot, c, t);
  return LWSE_OK;
}

// The earlier form of the tick: no patches, no placement, results copied to the caller's arrays.
LWSE_API int lwse_resident_sweep(lwse_engine* e, uint32_t flags, lwse_changes* ch) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  if (ch && ((ch->lws_capacity && (!ch->lws_rows || !ch->lws_out)) || (ch->group_capacity && (!ch->group_rows || !ch->group_out))))
    return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  TickCounts c;
  uint32_t slot = 0;
  int rc = drain_ticks_locked(e);
  if (rc == LWSE_OK) rc = tick_submit_locked(e, nullptr, 0, flags & LWSE_SWEEP_GANG);
  if (rc == LWSE_OK) rc = tick_wait_locked(e, &c, &slot);
  if (rc != LWSE_OK || !ch) return rc;
  ch->n_lws = c.n_lws;
  ch->n_groups = c.n_groups;
  const uint32_t nl = c.n_lws < ch->lws_capacity ? c.n_lws : ch->lws_capacity;
  const uint32_t ng = c.n_groups < ch->group_capacity ? c.n_groups : ch->group_capacity;
  const uint8_t* base = static_cast<const uint8_t*>(e->chg.h) + slot * e->chg_bytes;
  if (nl) {
    memcpy(ch->lws_rows, base + e->chg_off[0], (size_t)nl * 4);
    memcpy(ch->lws_out, base + e->chg_off[1], (size_t)nl * sizeof(lwse_lws_out));
  }
  if (ng) {
    memcpy(ch->group_rows, base + e->chg_off[2], (size_t)ng * 4);
    memcpy(ch->group_out, base + e->chg_off[3], (size_t)ng * sizeof(lwse_group_out));
  }
  return LWSE_OK;
}

LWSE_API int lwse_resident_place_outputs(lwse_engine* e, lwse_place_out* out) {
  if (!e || !out) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_place_loaded) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, cudaStreamSynchronize(e->side_stream));
  if (e->rn_reqs)
    LWSE_CUDA(e, cudaMemcpy(out, e->r_pout.p, (size_t)e->rn_reqs * sizeof(lwse_place_out), cudaMemcpyDeviceToHost));
  return LWSE_OK;
}

LWSE_API int lwse_resident_occupancy(lwse_engine* e, uint32_t* occupancy_out) {
  if (!e || !occupancy_out) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded || e->n_nodes == 0) return LWSE_ERR_NOT_READY;
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, cudaStreamSynchronize(e->stream));
  LWSE_CUDA(e, cudaMemcpy(occupancy_out, e->r_occ.p, (size_t)e->n_nodes * 4, cudaMemcpyDeviceToHost));
  return LWSE_OK;
}

LWSE_API int lwse_resident_tick_info(lwse_engine* e, lwse_tick_info* info) {
  if (!e || !info) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  *info = e->last_tick_info;
  return LWSE_OK;
}

LWSE_API int lwse_resident_node_info(lwse_engine* e, lwse_node_info* info) {
  if (!e || !info) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  *info = e->last_node_info;
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Placement what-if
// ---------------------------------------------------------------------------
// LWSE_WHATIF_TIMING=1: CUDA events around the device work of every what-if (lwse_debug_whatif_device_us)
static bool whatif_timing() {
  static const bool on = [] {
    const char* v = getenv("LWSE_WHATIF_TIMING");
    return v && atoi(v) != 0;
  }();
  return on;
}

// Every what-if runs on wf_stream behind an event on the engine's stream (the most recently submitted tick, both
// branches joined), reading the resident tables and the baseline results in place: nothing writes them while
// the call holds the mutex, and the call synchronizes its stream before it returns.
static int drain_begin_locked(lwse_engine* e) {
  LWSE_CUDA(e, e->wf_stream.ensure(cudaStreamNonBlocking));
  LWSE_CUDA(e, e->ev_wf.ensure(cudaEventDisableTiming));
  LWSE_CUDA(e, cudaEventRecord(e->ev_wf, e->stream));
  LWSE_CUDA(e, cudaStreamWaitEvent(e->wf_stream, e->ev_wf, 0));
  e->wf_timed = false;
  if (whatif_timing()) {
    LWSE_CUDA(e, e->ev_wf_t0.ensure(cudaEventDefault));
    LWSE_CUDA(e, e->ev_wf_t1.ensure(cudaEventDefault));
    LWSE_CUDA(e, cudaEventRecord(e->ev_wf_t0, e->wf_stream));
  }
  return LWSE_OK;
}

static int drain_end_locked(lwse_engine* e) {
  if (whatif_timing()) {
    LWSE_CUDA(e, cudaEventRecord(e->ev_wf_t1, e->wf_stream));
    e->wf_timed = true;
  }
  return LWSE_OK;
}

// The scratch of a private node index (wf_node_*), reserved before the snapshot: a reserve may reallocate.
static int reserve_node_index(lwse_engine* e) {
  LWSE_CUDA(e, e->wf_dom_first.reserve(((size_t)e->n_domains + 1) * 4 + 16));
  LWSE_CUDA(e, e->wf_node_order.reserve(((size_t)(e->n_nodes + 255u) / 256u + 1u) * 1024u + 16));
  LWSE_CUDA(e, e->wf_node_pos.reserve((size_t)e->n_nodes * 4 + 16));
  LWSE_CUDA(e, e->wf_node_ix.reserve(lwse::node_index_scratch_bytes(e->n_domains)));
  return LWSE_OK;
}

// A node index over `nodes` in the wf_node_* scratch, on s, for a what-if whose node rows the resident index
// does not describe; the index pointers are set to it (node_pos may be null).
static int own_node_index(lwse_engine* e, const lwse_node_rec* nodes, cudaStream_t s, const uint32_t** dom_first,
                          const uint32_t** node_order, const uint32_t** node_pos) {
  // The build wants its per-domain counts at zero.  A build leaves them so but not its cursors, and their
  // places move with n_domains (counts at [0, n), cursors at [n, 2n)): cleared before every build, as
  // lwse_upload_nodes clears the resident ones.  The padding of the order rows stays zero.
  LWSE_CUDA(e, cudaMemsetAsync(e->wf_node_ix.p, 0, lwse::node_index_scratch_bytes(e->n_domains), s));
  LWSE_CUDA(e, cudaMemsetAsync(e->wf_node_order.p, 0, ((size_t)(e->n_nodes + 255u) / 256u + 1u) * 1024u, s));
  LWSE_LAUNCH(e, lwse::launch_node_index(nodes, e->n_nodes, e->n_domains, (uint32_t*)e->wf_dom_first.p,
                                         (uint32_t*)e->wf_node_order.p, (uint32_t*)e->wf_node_pos.p, e->wf_node_ix.p,
                                         e->sm_count, s, false));
  *dom_first = (const uint32_t*)e->wf_dom_first.p;
  *node_order = (const uint32_t*)e->wf_node_order.p;
  if (node_pos) *node_pos = (const uint32_t*)e->wf_node_pos.p;
  return LWSE_OK;
}

// A what-if round (lwse_resident_place_whatif, lwse_resident_place_explain) in three steps: place_whatif_check
// (readiness, arguments, the touched namespaces and the node-index decision, over the host mirror), then
// place_whatif_reserve (its scratch: a reserve may reallocate, so before the snapshot), then, behind the snapshot
// event, place_whatif_enqueue (patched copies of the node and request rows in what-if scratch, the round over them
// on wf_stream, only the touched namespaces in the namespace form).  The resident node index is read in place
// unless the node patches need another one.
struct WhatifRound {
  const lwse_patch_seg* segs = nullptr;
  uint32_t n_segs = 0;
  const lwse_place_req* extra = nullptr;
  uint32_t n_extra = 0;
  uint32_t n_ns = 0, rn = 0, n_total = 0, n_touched = 0;
  bool ns_form = false, node_rows = false, node_rebuild = false, round_fresh = false;
  size_t stage_need = 0, round_bytes = 0;
  std::vector<uint8_t> touched;
  // the round's tables, once enqueued
  const lwse_node_rec* nodes = nullptr;
  const lwse_place_req* reqs = nullptr;
  lwse_place_out* out = nullptr;
};

// `bad_buffers`: the caller's own buffers are missing (refused as INVALID_ARG, after readiness).
static int place_whatif_check(lwse_engine* e, const lwse_patch_seg* segs, uint32_t n_segs, const lwse_place_req* extra,
                              uint32_t n_extra, uint32_t n_namespaces, bool bad_buffers, WhatifRound* w) {
  if (!e->r_loaded || !e->r_place_loaded || !e->r_place_current || e->n_nodes == 0 || e->n_domains == 0)
    return LWSE_ERR_NOT_READY;
  if (e->xch_world > 0) return LWSE_ERR_UNSUPPORTED;
  if ((n_segs && !segs) || n_segs > LWSE_TICK_MAX_SEGS || (n_extra && !extra) || bad_buffers) return LWSE_ERR_INVALID_ARG;
  const uint32_t n_ns = n_namespaces ? n_namespaces : e->rn_namespaces;
  if (n_ns == 0) return LWSE_ERR_INVALID_ARG;
  const uint32_t rn = e->rn_reqs;
  if ((uint64_t)rn + n_extra >= (1ull << 24)) return LWSE_ERR_UNSUPPORTED;
  for (uint32_t i = 0; i < n_segs; i++)
    if (segs[i].n && segs[i].table != LWSE_TABLE_NODES && segs[i].table != LWSE_TABLE_PLACE_REQS)
      return LWSE_ERR_INVALID_ARG;
  SegSummary ss;
  if (const int crc = summarize_segments(e, segs, n_segs, &ss); crc != LWSE_OK) return crc;
  // the node-index decision is the tick's, over the mirror, which stays as it is; then the touched namespaces
  const bool node_rows = (ss.tables & (1u << LWSE_TABLE_NODES)) != 0;
  bool node_rebuild = ss.node_moves;
  std::vector<uint8_t> touched(n_ns, 0);
  for (uint32_t v = e->rn_namespaces; v < n_ns; v++) touched[v] = 1;  // (their resident rows were UNSCHEDULABLE)
  size_t stage_need = align256((size_t)n_ns) + align256((size_t)n_extra * sizeof(lwse_place_req));
  for (uint32_t i = 0; i < n_segs; i++) {
    const lwse_patch_seg& g = segs[i];
    if (g.n == 0) continue;
    const bool range = (g.flags & LWSE_PATCH_RANGE) != 0;
    const uint32_t rb = g.table == LWSE_TABLE_NODES ? (uint32_t)sizeof(lwse_node_rec) : (uint32_t)sizeof(lwse_place_req);
    const uint32_t n_rows = g.table == LWSE_TABLE_NODES ? e->n_nodes : rn;
    stage_need += align256((size_t)g.n * 4) + align256((size_t)g.n * rb);
    for (uint32_t k = 0; k < g.n; k++) {
      const uint32_t row = range ? g.first_row + k : g.rows[k];
      if (row >= n_rows) return LWSE_ERR_INVALID_ARG;
      if (g.table == LWSE_TABLE_PLACE_REQS) {
        const uint32_t nv = static_cast<const lwse_place_req*>(g.values)[k].ns, ov = e->r_req_ns[row];
        if (nv < n_ns) touched[nv] = 1;
        if (ov < n_ns) touched[ov] = 1;
      }
    }
  }
  for (uint32_t i = 0; i < n_extra; i++)
    if (extra[i].ns < n_ns) touched[extra[i].ns] = 1;
  if (node_rows) std::fill(touched.begin(), touched.end(), (uint8_t)1);  // (capacities or domains moved under every namespace)
  // (a resident index behind the resident rows — node patches, and no round since because the request table is
  // empty — is not read either: the what-if builds its own)
  if (e->node_index_stale) node_rebuild = true;
  uint32_t n_touched = 0;
  for (uint8_t t : touched) n_touched += t;
  w->segs = segs;
  w->n_segs = n_segs;
  w->extra = extra;
  w->n_extra = n_extra;
  w->n_ns = n_ns;
  w->rn = rn;
  w->n_total = rn + n_extra;
  w->n_touched = n_touched;
  w->node_rows = node_rows;
  w->node_rebuild = node_rebuild;
  w->stage_need = stage_need;
  w->touched = std::move(touched);
  return LWSE_OK;
}

static int place_whatif_reserve(lwse_engine* e, WhatifRound* w) {
  // staging (the previous call synchronized its stream: the buffer is free)
  LWSE_CUDA(e, e->wf_stage.reserve(w->stage_need));
  LWSE_CUDA(e, e->wf_words.reserve(64));
  w->ns_form = lwse::place_ns_supported(e->n_nodes, e->n_domains);
  LWSE_CUDA(e, e->wf_reqs.reserve((size_t)w->n_total * sizeof(lwse_place_req) + 16));
  LWSE_CUDA(e, e->wf_out.reserve((size_t)w->n_total * sizeof(lwse_place_out) + 16));
  LWSE_CUDA(e, e->wf_touched.reserve((size_t)w->n_ns + 16));
  if (w->node_rows) LWSE_CUDA(e, e->wf_nodes.reserve((size_t)e->n_nodes * sizeof(lwse_node_rec) + 16));
  if (w->node_rebuild)
    if (const int rc = reserve_node_index(e); rc != LWSE_OK) return rc;
  if (w->ns_form) {
    w->round_bytes = lwse::place_ns_scratch_bytes(e->n_nodes, e->n_domains, w->n_total, w->n_ns);
    const void* before = e->wf_round.p;
    LWSE_CUDA(e, e->wf_round.reserve(w->round_bytes));
    // wf_geometry names the layout the scratch holds zeroed counts for: a new buffer holds none until
    // place_whatif_enqueue has cleared it, so a call that fails in between leaves the next one fresh
    if (before != e->wf_round.p) memset(e->wf_geometry, 0, sizeof(e->wf_geometry));
    const uint32_t geometry[4] = {w->n_total, w->n_ns, e->n_nodes, e->n_domains};
    w->round_fresh = memcmp(geometry, e->wf_geometry, sizeof(geometry)) != 0;
  } else {
    w->round_bytes = lwse::place_scratch_bytes(e->n_nodes, e->n_domains, w->n_total, w->n_ns);
    LWSE_CUDA(e, e->wf_round.reserve(w->round_bytes));
    e->wf_geometry[0] = e->wf_geometry[1] = e->wf_geometry[2] = e->wf_geometry[3] = 0;  // (the general form re-initialises it)
  }
  return LWSE_OK;
}

// On wf_stream, behind drain_begin_locked.
static int place_whatif_enqueue(lwse_engine* e, WhatifRound* w) {
  uint8_t* st_h = static_cast<uint8_t*>(e->wf_stage.h);
  size_t cursor = 0;
  auto stage = [&](const void* src, size_t bytes) -> size_t {
    const size_t at = cursor;
    if (bytes) memcpy(st_h + at, src, bytes);
    cursor += align256(bytes);
    return at;
  };
  cudaStream_t s = e->wf_stream;
  const uint32_t rn = w->rn, n_total = w->n_total, n_ns = w->n_ns;
  const size_t b_nodes = (size_t)e->n_nodes * sizeof(lwse_node_rec);
  lwse_node_rec* d_nodes = (lwse_node_rec*)e->nodes.p;
  lwse_place_req* d_reqs = (lwse_place_req*)e->wf_reqs.p;
  lwse_place_out* d_out = (lwse_place_out*)e->wf_out.p;
  if (w->node_rows) {
    LWSE_CUDA(e, cudaMemcpyAsync(e->wf_nodes.p, e->nodes.p, b_nodes, cudaMemcpyDeviceToDevice, s));
    d_nodes = (lwse_node_rec*)e->wf_nodes.p;
  }
  if (rn) {
    LWSE_CUDA(e, cudaMemcpyAsync(d_reqs, e->r_preq.p, (size_t)rn * sizeof(lwse_place_req), cudaMemcpyDeviceToDevice, s));
    LWSE_CUDA(e, cudaMemcpyAsync(d_out, e->r_pout.p, (size_t)rn * sizeof(lwse_place_out), cudaMemcpyDeviceToDevice, s));
  }
  if (w->n_extra) {
    const size_t at = stage(w->extra, (size_t)w->n_extra * sizeof(lwse_place_req));
    LWSE_CUDA(e, cudaMemcpyAsync(d_reqs + rn, st_h + at, (size_t)w->n_extra * sizeof(lwse_place_req), cudaMemcpyHostToDevice, s));
    LWSE_CUDA(e, cudaMemsetAsync(d_out + rn, 0, (size_t)w->n_extra * sizeof(lwse_place_out), s));
  }
  {
    const size_t at = stage(w->touched.data(), n_ns);
    LWSE_CUDA(e, cudaMemcpyAsync(e->wf_touched.p, st_h + at, n_ns, cudaMemcpyHostToDevice, s));
  }
  // the segments, into the copies: ranges by DMA first, then one scatter of the rest (as a tick applies them)
  lwse::ScatterSegHost sc[LWSE_TICK_MAX_SEGS];
  int n_sc = 0;
  for (uint32_t i = 0; i < w->n_segs; i++) {
    const lwse_patch_seg& g = w->segs[i];
    if (g.n == 0) continue;
    const bool is_nodes = g.table == LWSE_TABLE_NODES;
    const uint32_t rb = is_nodes ? (uint32_t)sizeof(lwse_node_rec) : (uint32_t)sizeof(lwse_place_req);
    void* table = is_nodes ? (void*)d_nodes : (void*)d_reqs;
    const size_t vat = stage(g.values, (size_t)g.n * rb);
    if (g.flags & LWSE_PATCH_RANGE) {
      LWSE_CUDA(e, cudaMemcpyAsync(static_cast<uint8_t*>(table) + (size_t)g.first_row * rb, st_h + vat, (size_t)g.n * rb,
                                   cudaMemcpyHostToDevice, s));
      continue;
    }
    const size_t rat = stage(g.rows, (size_t)g.n * 4);
    uint8_t* st_d = static_cast<uint8_t*>(e->wf_stage.d);
    sc[n_sc++] = lwse::ScatterSegHost{table, is_nodes ? (uint64_t)e->n_nodes : (uint64_t)rn,
                                      reinterpret_cast<const uint32_t*>(st_d + rat), st_d + vat, g.n, rb, false};
  }
  if (n_sc) {
    LWSE_LAUNCH(e, lwse::launch_scatter(sc, n_sc, nullptr, 0, s, false));
  }
  const uint32_t* dom_first = (const uint32_t*)e->dom_first.p;
  const uint32_t* node_order = (const uint32_t*)e->node_order.p;
  const uint32_t* node_pos = (const uint32_t*)e->node_pos.p;
  if (w->node_rebuild)
    if (const int rc = own_node_index(e, d_nodes, s, &dom_first, &node_order, &node_pos); rc != LWSE_OK) return rc;
  if (w->ns_form) {
    if (w->round_fresh) {  // (index counts and counters start at zero)
      LWSE_CUDA(e, cudaMemsetAsync(e->wf_round.p, 0, w->round_bytes, s));
      const uint32_t geometry[4] = {n_total, n_ns, e->n_nodes, e->n_domains};
      memcpy(e->wf_geometry, geometry, sizeof(geometry));
    }
    LWSE_LAUNCH(e, lwse::launch_place_whatif_index(d_reqs, n_total, n_ns, (const uint8_t*)e->wf_touched.p, e->n_nodes, e->n_domains,
                                                   e->wf_round.p, e->sm_count, s));
    LWSE_LAUNCH(e, lwse::launch_place_ns(d_nodes, dom_first, node_order, e->n_nodes, e->n_domains, d_reqs, n_total,
                                         (const uint32_t*)e->r_occ.p, 1, 0, n_ns, d_out, e->wf_round.p, w->round_bytes, false,
                                         e->wf_calls++, false, e->sm_count, s, nullptr, false, nullptr, nullptr,
                                         lwse::kNsIndexReuse));
  } else {
    LWSE_LAUNCH(e, lwse::launch_place(d_nodes, dom_first, node_order, node_pos, e->n_nodes, e->n_domains, d_reqs, n_total,
                                      (const uint32_t*)e->r_occ.p, n_ns, d_out, e->wf_round.p, w->round_bytes, nullptr,
                                      e->sm_count, s, 0u, true, 1, n_total, 0, nullptr, nullptr, nullptr, false));
  }
  w->nodes = d_nodes;
  w->reqs = d_reqs;
  w->out = d_out;
  return LWSE_OK;
}

// The what-if round, then one diff kernel against the baseline rows (r_pout, read in place: nothing writes them
// while the call holds the mutex).
LWSE_API int lwse_resident_place_whatif(lwse_engine* e, lwse_place_whatif* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  WhatifRound w;
  const bool bad_buffers = (q->n_extra && !q->extra_out) || (q->capacity && (!q->rows || !q->before || !q->after));
  if (const int rc = place_whatif_check(e, q->segs, q->n_segs, q->extra, q->n_extra, q->n_namespaces, bad_buffers, &w);
      rc != LWSE_OK)
    return rc;
  const uint32_t rn = w.rn, n_total = w.n_total;

  DeviceGuard guard(e->device);
  const uint32_t list_cap = q->capacity < rn ? q->capacity : rn;  // (at most rn rows can differ)
  LWSE_CUDA(e, e->wf_list.reserve(64 + 16 + (size_t)list_cap * (4 + 2 * sizeof(lwse_place_out))));
  if (const int rc = place_whatif_reserve(e, &w); rc != LWSE_OK) return rc;

  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  if (const int rc = place_whatif_enqueue(e, &w); rc != LWSE_OK) return rc;
  lwse_place_out* d_out = w.out;
  // the diff against the baseline, the counts
  // (layout: [counts: 16 words] [rows: list_cap] [before: list_cap] [after: list_cap], the 16-byte rows aligned)
  uint32_t* d_counts = (uint32_t*)e->wf_list.p;
  uint32_t* d_rows = d_counts + 16;
  lwse_place_out* d_before =
      reinterpret_cast<lwse_place_out*>(static_cast<uint8_t*>(e->wf_list.p) + 64 + (((size_t)list_cap * 4 + 15) & ~(size_t)15));
  lwse_place_out* d_after = d_before + list_cap;
  LWSE_CUDA(e, cudaMemsetAsync(d_counts, 0, 64, s));
  {
    LWSE_LAUNCH(e, lwse::launch_place_whatif_diff((const lwse_place_out*)e->r_pout.p, d_out, rn, n_total, d_rows, d_before,
                                                  d_after, list_cap, d_counts, e->sm_count, s));
  }
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_counts, 32, cudaMemcpyDeviceToHost, s));
  if (q->n_extra)
    LWSE_CUDA(e, cudaMemcpyAsync(q->extra_out, d_out + rn, (size_t)q->n_extra * sizeof(lwse_place_out), cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint32_t n_changed = words[0];
  const uint32_t listed = n_changed < list_cap ? n_changed : list_cap;
  if (listed) {
    LWSE_CUDA(e, cudaMemcpyAsync(q->rows, d_rows, (size_t)listed * 4, cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaMemcpyAsync(q->before, d_before, (size_t)listed * sizeof(lwse_place_out), cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaMemcpyAsync(q->after, d_after, (size_t)listed * sizeof(lwse_place_out), cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaStreamSynchronize(s));
  }
  q->n_changed = n_changed;
  q->n_lost = words[1];
  q->n_moved = words[2];
  q->n_gained = words[3];
  q->n_placed = words[4];
  q->n_unschedulable = words[5];
  q->n_conflict = words[6];
  q->namespaces_solved = w.ns_form ? w.n_touched : 0u;
  q->form = w.ns_form ? LWSE_TICK_FORM_NAMESPACE : LWSE_TICK_FORM_GENERAL;
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Placement explanation
// ---------------------------------------------------------------------------
// The round is the baseline (r_pout over the resident node and request rows, read in place) or the what-if's (the
// what-if's check, reserve and enqueue steps); launch_place_explain runs over it on wf_stream, behind the same
// snapshot event, with scratch of its own (px_*).
static uint64_t table_slots(uint64_t pairs);
LWSE_API int lwse_resident_place_explain(lwse_engine* e, lwse_place_explain_query* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  WhatifRound w;
  const bool bad_buffers = (q->n_rows && !q->rows) || (q->capacity && !q->out);
  if (const int rc = place_whatif_check(e, q->segs, q->n_segs, q->extra, q->n_extra, q->n_namespaces, bad_buffers, &w);
      rc != LWSE_OK)
    return rc;
  const bool whatif = q->n_segs || q->n_extra || w.n_ns != e->rn_namespaces;
  const bool by_mask = q->rows == nullptr;
  const uint32_t n_total = w.n_total, nd = e->n_domains;
  if (!by_mask)
    for (uint32_t i = 0; i < q->n_rows; i++)
      if (q->rows[i] >= n_total) return LWSE_ERR_INVALID_ARG;
  const uint32_t n_listed = by_mask ? n_total : q->n_rows;
  const uint32_t out_cap = q->capacity < n_listed ? q->capacity : n_listed;
  const uint32_t n_chunks = by_mask ? (n_total + 255u) / 256u : 0u;
  const uint64_t slots = table_slots(n_total);

  DeviceGuard guard(e->device);
  if (whatif)
    if (const int rc = place_whatif_reserve(e, &w); rc != LWSE_OK) return rc;
  // px_sel: [the listed count, 3 words of padding] [chunk count | first | cursor] [the list]
  const size_t sel_words = 4 + (size_t)3 * n_chunks + 1 + n_listed;
  LWSE_CUDA(e, e->px_sel.reserve(sel_words * 4 + 16));
  LWSE_CUDA(e, e->px_dom.reserve((size_t)3 * nd * 4 + 16));
  LWSE_CUDA(e, e->px_mark.reserve((size_t)w.n_ns + 16));
  LWSE_CUDA(e, e->px_table.reserve((size_t)slots * 16));
  LWSE_CUDA(e, e->px_out.reserve(128 + (size_t)out_cap * sizeof(lwse_place_explain_row)));
  LWSE_CUDA(e, e->px_host.reserve(256 + (by_mask ? 0 : (size_t)n_listed * 4)));

  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  lwse::PlaceExplainLaunch p{};
  if (whatif) {
    if (const int rc = place_whatif_enqueue(e, &w); rc != LWSE_OK) return rc;
    p.nodes = w.nodes;
    p.reqs = w.reqs;
    p.res = w.out;
  } else {
    p.nodes = (const lwse_node_rec*)e->nodes.p;
    p.reqs = (const lwse_place_req*)e->r_preq.p;
    p.res = (const lwse_place_out*)e->r_pout.p;
  }
  uint32_t* sel = (uint32_t*)e->px_sel.p;
  uint32_t* h_words = static_cast<uint32_t*>(e->px_host.h);
  p.occupancy = (const uint32_t*)e->r_occ.p;
  p.n_nodes = e->n_nodes;
  p.n_domains = nd;
  p.n_rows = n_total;
  p.n_namespaces = w.n_ns;
  p.by_mask = by_mask;
  p.mask = q->mask;
  p.chunk_count = sel + 4;
  p.chunk_first = p.chunk_count + n_chunks;
  p.chunk_cursor = p.chunk_first + n_chunks + 1;
  p.list = p.chunk_cursor + n_chunks;
  p.n_list = by_mask ? p.chunk_first + n_chunks : sel;
  p.n_listed = n_listed;
  p.dom = (uint32_t*)e->px_dom.p;
  p.ns_mark = (uint8_t*)e->px_mark.p;
  p.tkeys = (unsigned long long*)e->px_table.p;
  p.tvals = p.tkeys + slots;
  p.table_mask = (uint32_t)(slots - 1);
  p.totals = (unsigned long long*)e->px_out.p;
  p.out = reinterpret_cast<lwse_place_explain_row*>(static_cast<uint8_t*>(e->px_out.p) + 128);
  p.capacity = out_cap;
  if (!by_mask) {  // the caller's rows, behind their count (px_host: the previous call synchronized its stream)
    h_words[0] = n_listed;
    if (n_listed) memcpy(h_words + 64, q->rows, (size_t)n_listed * 4);
    LWSE_CUDA(e, cudaMemcpyAsync(sel, h_words, 4, cudaMemcpyHostToDevice, s));
    if (n_listed) LWSE_CUDA(e, cudaMemcpyAsync(p.list, h_words + 64, (size_t)n_listed * 4, cudaMemcpyHostToDevice, s));
  }
  LWSE_CUDA(e, cudaMemsetAsync(p.dom, 0, (size_t)3 * nd * 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(p.ns_mark, 0, w.n_ns, s));
  LWSE_CUDA(e, cudaMemsetAsync(p.tkeys, 0xFF, (size_t)slots * 16, s));
  LWSE_CUDA(e, cudaMemsetAsync(p.totals, 0, 128, s));
  LWSE_LAUNCH(e, lwse::launch_place_explain(&p, e->sm_count, s));
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  // read back: the totals and the listed count, then the rows
  unsigned long long* h_totals = reinterpret_cast<unsigned long long*>(h_words);
  LWSE_CUDA(e, cudaMemcpyAsync(h_totals, p.totals, 128, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(h_words + 32, p.n_list, 4, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint32_t n_explained = h_words[32];
  const uint32_t listed = n_explained < out_cap ? n_explained : out_cap;
  if (listed) {
    LWSE_CUDA(e, cudaMemcpyAsync(q->out, p.out, (size_t)listed * sizeof(lwse_place_explain_row), cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaStreamSynchronize(s));
  }
  q->n_explained = n_explained;
  q->round_rows = n_total;
  q->n_domains = nd;
  q->whatif = whatif ? 1u : 0u;
  q->form = whatif ? (w.ns_form ? LWSE_TICK_FORM_NAMESPACE : LWSE_TICK_FORM_GENERAL) : 0u;
  for (uint32_t b = 0; b < 7; b++) q->n_flag[b] = (uint32_t)h_totals[8 + b];
  for (uint32_t j = 0; j < 8; j++) q->n_class[j] = h_totals[j];
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Drain what-if and drain cost
// ---------------------------------------------------------------------------
// The restart walk over the resident tables (the drain budget's passes and the pair walk), its key rows in `cost`
// and its counters at `counts`.
static lwse::DrainBudgetCostLaunch restart_walk(const lwse_engine* e, bool by_domain, lwse_drain_budget_cost* cost,
                                                uint32_t* counts) {
  lwse::DrainBudgetCostLaunch p{};
  p.lws = (const lwse_lws_rec*)e->r_lws.p;
  p.lws_out = (const lwse_lws_out*)e->r_lws_out.p;
  p.groups = (const lwse_group_rec*)e->r_groups.p;
  p.pod_state = (const uint8_t*)e->r_pst.p;
  p.pod_ident = (const lwse_pod_ident*)e->r_pid.p;
  p.baseline = (const lwse_group_out*)e->r_group_out.p;
  p.nodes = (const lwse_node_rec*)e->nodes.p;
  p.occupancy = (const uint32_t*)e->r_occ.p;
  p.cost = cost;
  p.counts = counts;
  p.n_pods = e->rn_pods;
  p.n_lws = e->rn_lws;
  p.n_groups = e->rn_groups;
  p.n_nodes = e->n_nodes;
  p.n_domains = e->n_domains;
  p.n_keys = by_domain ? e->n_domains : e->n_nodes;
  p.by_domain = by_domain;
  return p;
}

// The slots of a linear-probing table for `pairs` entries: a power of two at least twice their count, so a probe
// always finds a free slot, and at least 256.
static uint64_t table_slots(uint64_t pairs) {
  uint64_t slots = 256;
  while (slots < 2 * pairs) slots <<= 1;
  return slots;
}

// The query's m keys are distinct and below nk (marked in wf_stage's host side: before the snapshot, so nothing
// in flight reads it).
static int check_key_ids(lwse_engine* e, const uint32_t* ids, uint32_t m, uint32_t nk) {
  LWSE_CUDA(e, e->wf_stage.reserve((size_t)nk + 16));
  uint8_t* seen = static_cast<uint8_t*>(e->wf_stage.h);
  memset(seen, 0, nk);
  for (uint32_t i = 0; i < m; i++) {
    if (ids[i] >= nk || seen[ids[i]]) return LWSE_ERR_INVALID_ARG;  // out of range, or a duplicate
    seen[ids[i]] = 1;
  }
  return LWSE_OK;
}

// The scratch of the what-if's sweep (lwse_resident_drain_whatif and the set form of the drain budget).
static int reserve_drain_sweep(lwse_engine* e) {
  const uint32_t ng = e->rn_groups;
  const uint64_t np = e->rn_pods;
  LWSE_CUDA(e, e->wf_stage.reserve((size_t)e->n_nodes));  // (the previous what-if synchronized its stream: free)
  LWSE_CUDA(e, e->wf_words.reserve(64));
  LWSE_CUDA(e, e->dr_state.reserve((size_t)np + 16));
  LWSE_CUDA(e, e->dr_groups.reserve((size_t)ng * sizeof(lwse_group_rec) + 16));
  LWSE_CUDA(e, e->dr_out.reserve((size_t)ng * sizeof(lwse_group_out) + 16));
  LWSE_CUDA(e, e->dr_scan.reserve(lwse::lws_sweep_scratch_bytes(np, ng)));
  LWSE_CUDA(e, e->dr_mask.reserve((size_t)e->n_nodes + 16));
  return LWSE_OK;
}

// Copies of the state column and the group rows, the mark kernel on them (the node mask in dr_mask), the
// sweep's group pass over {resident LWS rows, copied groups, copied states, resident identity rows} into
// dr_out (the LWS pass is skipped: it reads only flag bits eviction does not change), then the diff against
// the baseline; on wf_stream, after the caller zeroed the 16 counters at d_counts.
static int enqueue_drain_sweep(lwse_engine* e, uint32_t* d_counts, uint32_t* d_rows, lwse_group_out* d_before,
                               lwse_group_out* d_after, uint32_t list_cap) {
  const uint32_t ng = e->rn_groups, nn = e->n_nodes;
  const uint64_t np = e->rn_pods;
  cudaStream_t s = e->wf_stream;
  if (np) LWSE_CUDA(e, cudaMemcpyAsync(e->dr_state.p, e->r_pst.p, (size_t)np, cudaMemcpyDeviceToDevice, s));
  if (ng) LWSE_CUDA(e, cudaMemcpyAsync(e->dr_groups.p, e->r_groups.p, (size_t)ng * sizeof(lwse_group_rec), cudaMemcpyDeviceToDevice, s));
  LWSE_LAUNCH(e, lwse::launch_drain_mark((const uint8_t*)e->dr_mask.p, nn, (const lwse_pod_ident*)e->r_pid.p, (uint8_t*)e->dr_state.p,
                                         np, (lwse_group_rec*)e->dr_groups.p, ng, d_counts, e->sm_count, s));
  lwse_lws_tables d{};
  d.lws = (const lwse_lws_rec*)e->r_lws.p;
  d.n_lws = e->rn_lws;
  d.groups = (const lwse_group_rec*)e->dr_groups.p;
  d.n_groups = ng;
  d.pod_state = (const lwse_pod_state*)e->dr_state.p;
  d.pod_ident = (const lwse_pod_ident*)e->r_pid.p;
  d.n_pods = np;
  d.group_out = (lwse_group_out*)e->dr_out.p;
  d.flags = e->r_sweep_flags | LWSE_SWEEP_SKIP_LWS_PASS;
  LWSE_LAUNCH(e, lwse::launch_lws_sweep(&d, (const lwse_node_rec*)e->nodes.p, nn, e->dr_scan.p, e->sm_count, s, nullptr,
                                        nullptr, /*first_mode=*/0));
  return count_launch(e, lwse::launch_drain_diff((const lwse_group_out*)e->r_group_out.p, (const lwse_group_out*)e->dr_out.p,
                                                 (const lwse_group_rec*)e->r_groups.p, ng, d_rows, d_before, d_after, list_cap, d_counts,
                                                 e->sm_count, s));
}

LWSE_API int lwse_resident_drain_whatif(lwse_engine* e, lwse_drain_whatif* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded || e->n_nodes == 0 || !e->r_groups_swept) return LWSE_ERR_NOT_READY;
  if ((q->n_nodes && !q->nodes) || (q->capacity && (!q->rows || !q->before || !q->after))) return LWSE_ERR_INVALID_ARG;
  for (uint32_t i = 0; i < q->n_nodes; i++)
    if (q->nodes[i] >= e->n_nodes) return LWSE_ERR_INVALID_ARG;
  const uint32_t ng = e->rn_groups, nn = e->n_nodes;
  const uint32_t list_cap = q->capacity < ng ? q->capacity : ng;  // (at most ng rows can differ)
  DeviceGuard guard(e->device);
  if (const int rc = reserve_drain_sweep(e); rc != LWSE_OK) return rc;
  // (layout: [counts: 16 words] [rows: list_cap] [before: list_cap] [after: list_cap], the 16-byte rows aligned)
  const size_t rows_bytes = ((size_t)list_cap * 4 + 15) & ~(size_t)15;
  LWSE_CUDA(e, e->dr_list.reserve(64 + rows_bytes + (size_t)list_cap * 2 * sizeof(lwse_group_out)));
  uint8_t* mask = static_cast<uint8_t*>(e->wf_stage.h);
  memset(mask, 0, nn);
  for (uint32_t i = 0; i < q->n_nodes; i++) mask[q->nodes[i]] = 1;
  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* d_counts = (uint32_t*)e->dr_list.p;
  uint32_t* d_rows = d_counts + 16;
  lwse_group_out* d_before = reinterpret_cast<lwse_group_out*>(static_cast<uint8_t*>(e->dr_list.p) + 64 + rows_bytes);
  lwse_group_out* d_after = d_before + list_cap;
  LWSE_CUDA(e, cudaMemcpyAsync(e->dr_mask.p, mask, nn, cudaMemcpyHostToDevice, s));
  LWSE_CUDA(e, cudaMemsetAsync(d_counts, 0, 64, s));
  if (const int rc = enqueue_drain_sweep(e, d_counts, d_rows, d_before, d_after, list_cap); rc != LWSE_OK) return rc;
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_counts, 32, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint32_t n_changed = words[0];
  const uint32_t listed = n_changed < list_cap ? n_changed : list_cap;
  if (listed) {
    LWSE_CUDA(e, cudaMemcpyAsync(q->rows, d_rows, (size_t)listed * 4, cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaMemcpyAsync(q->before, d_before, (size_t)listed * sizeof(lwse_group_out), cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaMemcpyAsync(q->after, d_after, (size_t)listed * sizeof(lwse_group_out), cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaStreamSynchronize(s));
  }
  q->n_changed = n_changed;
  q->n_pods_evicted = words[1];
  q->n_leaders_evicted = words[2];
  q->n_groups_restarted = words[3];
  q->n_ready_restarted = words[4];
  uint64_t recreated = 0;
  memcpy(&recreated, words + 6, 8);
  q->n_pods_recreated = recreated;
  return LWSE_OK;
}

// Every node in one pass: the rows start as {pods = the resident occupancy counter, zeros}, then
// drain_cost_kernel adds each group's restart to the nodes it would restart from.
LWSE_API int lwse_resident_drain_cost(lwse_engine* e, lwse_drain_cost* out) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded || e->n_nodes == 0 || !e->r_groups_swept) return LWSE_ERR_NOT_READY;
  if (!out) return LWSE_ERR_INVALID_ARG;
  const uint32_t nn = e->n_nodes;
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, e->dr_cost.reserve((size_t)nn * sizeof(lwse_drain_cost) + 16));
  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  lwse_drain_cost* d_cost = (lwse_drain_cost*)e->dr_cost.p;
  LWSE_CUDA(e, cudaMemsetAsync(d_cost, 0, (size_t)nn * sizeof(lwse_drain_cost), s));
  LWSE_CUDA(e, cudaMemcpy2DAsync(d_cost, sizeof(lwse_drain_cost), e->r_occ.p, 4, 4, nn, cudaMemcpyDeviceToDevice, s));
  LWSE_LAUNCH(e, lwse::launch_drain_cost((const lwse_lws_rec*)e->r_lws.p, e->rn_lws, (const lwse_group_rec*)e->r_groups.p,
                                         e->rn_groups, (const uint8_t*)e->r_pst.p, (const lwse_pod_ident*)e->r_pid.p,
                                         e->rn_pods, (const lwse_group_out*)e->r_group_out.p, d_cost, nn, e->sm_count, s));
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(out, d_cost, (size_t)nn * sizeof(lwse_drain_cost), cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Drain budget
// ---------------------------------------------------------------------------
static bool drain_budget_ready(const lwse_engine* e) {
  return e->r_loaded && e->n_nodes != 0 && e->r_groups_swept && e->r_swept;
}

// The node mask of a drain set in dr_mask, on wf_stream: `mask` (host) marks node rows, or domain ids whose
// nodes the device marks.
static int enqueue_drain_set(lwse_engine* e, const uint8_t* mask, bool by_domain) {
  const uint32_t nn = e->n_nodes, nd = e->n_domains;
  cudaStream_t s = e->wf_stream;
  if (!by_domain) {
    LWSE_CUDA(e, cudaMemcpyAsync(e->dr_mask.p, mask, nn, cudaMemcpyHostToDevice, s));
    return LWSE_OK;
  }
  if (nd) LWSE_CUDA(e, cudaMemcpyAsync(e->dr_domains.p, mask, nd, cudaMemcpyHostToDevice, s));
  return count_launch(e, lwse::launch_drain_domain_mask((const uint8_t*)e->dr_domains.p, nd, (const lwse_node_rec*)e->nodes.p, nn,
                                                        (uint8_t*)e->dr_mask.p, e->sm_count, s));
}

// The set form: the drain what-if's sweep over the node mask (the given node rows, or the nodes of the given
// domains, built on the device), the diff's totals without a change list, then drain_budget_kernel over
// every LWS row.
LWSE_API int lwse_resident_drain_budget(lwse_engine* e, lwse_drain_budget_query* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!drain_budget_ready(e)) return LWSE_ERR_NOT_READY;
  if (q->scope != LWSE_DRAIN_NODES && q->scope != LWSE_DRAIN_DOMAINS) return LWSE_ERR_INVALID_ARG;
  if ((q->n_ids && !q->ids) || (q->capacity && !q->rows)) return LWSE_ERR_INVALID_ARG;
  const bool by_domain = q->scope == LWSE_DRAIN_DOMAINS;
  const uint32_t nn = e->n_nodes, nd = e->n_domains, n_keys = by_domain ? nd : nn;
  for (uint32_t i = 0; i < q->n_ids; i++)
    if (q->ids[i] >= n_keys) return LWSE_ERR_INVALID_ARG;
  const uint32_t nl = e->rn_lws;
  const uint32_t list_cap = q->capacity < nl ? q->capacity : nl;
  DeviceGuard guard(e->device);
  if (const int rc = reserve_drain_sweep(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, e->wf_stage.reserve((size_t)n_keys));
  LWSE_CUDA(e, e->dr_list.reserve(64));
  LWSE_CUDA(e, e->dr_brows.reserve((size_t)list_cap * sizeof(lwse_drain_budget) + 16));
  if (by_domain) LWSE_CUDA(e, e->dr_domains.reserve((size_t)nd + 16));
  uint8_t* mask = static_cast<uint8_t*>(e->wf_stage.h);
  memset(mask, 0, n_keys);
  for (uint32_t i = 0; i < q->n_ids; i++) mask[q->ids[i]] = 1;
  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* d_counts = (uint32_t*)e->dr_list.p;
  lwse_drain_budget* d_rows = (lwse_drain_budget*)e->dr_brows.p;
  if (const int rc = enqueue_drain_set(e, mask, by_domain); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemsetAsync(d_counts, 0, 64, s));
  if (const int rc = enqueue_drain_sweep(e, d_counts, nullptr, nullptr, nullptr, 0); rc != LWSE_OK) return rc;
  LWSE_LAUNCH(e, lwse::launch_drain_budget((const lwse_lws_rec*)e->r_lws.p, (const lwse_lws_out*)e->r_lws_out.p, nl,
                                           (const lwse_group_rec*)e->r_groups.p, (const lwse_group_out*)e->r_group_out.p,
                                           (const lwse_group_out*)e->dr_out.p, e->rn_groups, d_rows, list_cap, d_counts,
                                           e->sm_count, s));
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_counts, 64, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint32_t n_touched = words[8];
  const uint32_t listed = n_touched < list_cap ? n_touched : list_cap;
  if (listed) {
    LWSE_CUDA(e, cudaMemcpyAsync(q->rows, d_rows, (size_t)listed * sizeof(lwse_drain_budget), cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaStreamSynchronize(s));
  }
  q->n_touched = n_touched;
  q->n_breached = words[9];
  q->n_loses_available = words[10];
  q->n_already_below = words[11];
  q->n_pods_evicted = words[1];
  q->n_leaders_evicted = words[2];
  q->n_groups_restarted = words[3];
  q->n_ready_restarted = words[4];
  uint64_t recreated = 0;
  memcpy(&recreated, words + 6, 8);
  q->n_pods_recreated = recreated;
  return LWSE_OK;
}

// The per-key form: the key rows and the pair count (pass 0), one host synchronisation to size the (LWS, key)
// table from that count (a power of two at least twice it, so linear probing always finds a slot), then the
// table and the key rows' budget columns (pass 1).
LWSE_API int lwse_resident_drain_budget_cost(lwse_engine* e, uint32_t scope, lwse_drain_budget_cost* out) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!drain_budget_ready(e)) return LWSE_ERR_NOT_READY;
  if (!out || (scope != LWSE_DRAIN_NODES && scope != LWSE_DRAIN_DOMAINS)) return LWSE_ERR_INVALID_ARG;
  const bool by_domain = scope == LWSE_DRAIN_DOMAINS;
  const uint32_t nn = e->n_nodes, n_keys = by_domain ? e->n_domains : nn;
  const size_t cost_bytes = (size_t)n_keys * sizeof(lwse_drain_budget_cost);
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, e->dr_bcost.reserve(cost_bytes + 16));
  LWSE_CUDA(e, e->dr_bwords.reserve(64));
  LWSE_CUDA(e, e->wf_words.reserve(64));
  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  lwse::DrainBudgetCostLaunch p = restart_walk(e, by_domain, (lwse_drain_budget_cost*)e->dr_bcost.p, (uint32_t*)e->dr_bwords.p);
  LWSE_CUDA(e, cudaMemsetAsync(p.cost, 0, cost_bytes, s));
  LWSE_CUDA(e, cudaMemsetAsync(p.counts, 0, 64, s));
  LWSE_LAUNCH(e, lwse::launch_drain_budget_cost(&p, 0, e->sm_count, s));
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  LWSE_CUDA(e, cudaMemcpyAsync(words, p.counts, 16, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  uint64_t pairs = 0;
  memcpy(&pairs, words, 8);
  if (pairs) {
    if (pairs > (1ull << 30)) return LWSE_ERR_OOM;  // (the table index is 32-bit)
    const uint64_t slots = table_slots(pairs);
    LWSE_CUDA(e, e->dr_table.reserve((size_t)slots * (sizeof(unsigned long long) + sizeof(uint4))));
    p.keys = (unsigned long long*)e->dr_table.p;
    p.vals = reinterpret_cast<uint4*>(p.keys + slots);
    p.table_mask = (uint32_t)(slots - 1);
    LWSE_CUDA(e, cudaMemsetAsync(p.keys, 0xFF, (size_t)slots * sizeof(unsigned long long), s));
    LWSE_CUDA(e, cudaMemsetAsync(p.vals, 0, (size_t)slots * sizeof(uint4), s));
    LWSE_LAUNCH(e, lwse::launch_drain_budget_cost(&p, 1, e->sm_count, s));
  }
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  if (n_keys) LWSE_CUDA(e, cudaMemcpyAsync(out, p.cost, cost_bytes, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words, p.counts, 16, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  if (words[2]) return LWSE_ERR_OOM;  // an insert the table refused: no answer rather than a wrong one
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Drain waves
// ---------------------------------------------------------------------------
// The drain waves chain up to its dense rows, shared by lwse_resident_drain_waves, lwse_resident_ds_drain_waves and
// lwse_resident_drain_place_waves.  Its steps enqueue on wf_stream and never synchronize.  The caller zeroes the
// counter blocks the steps write (one block may hold other counters too), issues every read-back, and launches
// passes 1 and 2, whose variant differs between the planners.

// A waves answer: the totals (16 B), m key rows, then max_waves wave rows.  (Templates over the query and row
// types, so with C++ linkage inside the API block.)
extern "C++" {
template <class Key, class Wave>
static size_t waves_answer_bytes(uint32_t m, uint32_t max_waves) {
  return 16 + (size_t)m * sizeof(Key) + (size_t)max_waves * sizeof(Wave);
}

// A waves answer, read back into dv_host by the caller's last synchronisation, copied out to the query.
template <class Q>
static void copy_waves_answer(const lwse_engine* e, Q* q) {
  const uint8_t* h = static_cast<const uint8_t*>(e->dv_host.h);
  const size_t keys_bytes = (size_t)q->n_ids * sizeof(*q->keys);
  uint32_t totals[4];
  memcpy(totals, h, 16);
  if (q->n_ids) memcpy(q->keys, h + 16, keys_bytes);
  memcpy(q->waves, h + 16 + keys_bytes, (size_t)totals[0] * sizeof(*q->waves));
  q->n_waves = totals[0];
  q->n_planned = totals[1];
  q->n_breaches_alone = totals[2];
  q->n_no_wave = totals[3];
}
}  // extern "C++"

// The chain's scratch for m keys out of nk, and dv_host, which carries the keys in and the caller's answer of
// answer_bytes out: reserved once at the larger size, before the snapshot.
static int reserve_drain_waves(lwse_engine* e, uint32_t m, uint32_t nk, uint32_t max_waves, size_t answer_bytes) {
  const uint32_t nl = e->rn_lws, ng = e->rn_groups;
  LWSE_CUDA(e, e->dv_ids.reserve((size_t)m * 4 + 16));
  LWSE_CUDA(e, e->dv_pos.reserve((size_t)nk * 4 + 16));
  LWSE_CUDA(e, e->dv_kidx.reserve(((size_t)m * 3 + 2) * 4 + 16));
  LWSE_CUDA(e, e->dv_lidx.reserve(((size_t)nl * 3 + 2) * 4 + 16));
  LWSE_CUDA(e, e->dv_dense.reserve((size_t)nl * 16 + 16));
  LWSE_CUDA(e, e->dv_gwaves.reserve((size_t)ng * 8 + 16));
  LWSE_CUDA(e, e->dv_out.reserve(waves_answer_bytes<lwse_drain_wave_key, lwse_drain_wave>(m, max_waves)));
  LWSE_CUDA(e, e->dv_host.reserve(std::max(answer_bytes, (size_t)m * 4)));
  return LWSE_OK;
}

// The keys in through dv_host, the chain's scratch and the walk's key rows zeroed, the restart walk's pass 0 (`bp`),
// then the chain's pass 0 into p, its counters at `counts`.
static int enqueue_drain_waves_setup(lwse_engine* e, const lwse::DrainBudgetCostLaunch& bp, const uint32_t* ids, uint32_t m,
                                     uint32_t max_waves, unsigned long long* counts, lwse::DrainWavesLaunch* p) {
  const uint32_t nl = e->rn_lws, ng = e->rn_groups, nk = bp.n_keys;
  cudaStream_t s = e->wf_stream;
  if (m) {
    memcpy(e->dv_host.h, ids, (size_t)m * 4);
    LWSE_CUDA(e, cudaMemcpyAsync(e->dv_ids.p, e->dv_host.h, (size_t)m * 4, cudaMemcpyHostToDevice, s));
  }
  LWSE_CUDA(e, cudaMemsetAsync(bp.cost, 0, (size_t)nk * sizeof(lwse_drain_budget_cost), s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dv_pos.p, 0xFF, (size_t)nk * 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dv_kidx.p, 0, (size_t)m * 4 + 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dv_lidx.p, 0, (size_t)nl * 4 + 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dv_gwaves.p, 0, (size_t)ng * 8, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dv_out.p, 0, waves_answer_bytes<lwse_drain_wave_key, lwse_drain_wave>(m, max_waves), s));
  LWSE_LAUNCH(e, lwse::launch_drain_budget_cost(&bp, 0, e->sm_count, s));
  p->lws = bp.lws;
  p->lws_out = bp.lws_out;
  p->groups = bp.groups;
  p->baseline = bp.baseline;
  p->cost = bp.cost;
  p->ids = (const uint32_t*)e->dv_ids.p;
  p->pos_of = (uint32_t*)e->dv_pos.p;
  p->count = (uint32_t*)e->dv_kidx.p;
  p->first = p->count + m;
  p->cursor = p->first + m + 1;
  p->l_count = (uint32_t*)e->dv_lidx.p;
  p->l_first = p->l_count + nl;
  p->l_cursor = p->l_first + nl + 1;
  p->dense = (uint4*)e->dv_dense.p;
  p->g_waves = (unsigned long long*)e->dv_gwaves.p;
  p->out = (uint8_t*)e->dv_out.p;
  p->counts = counts;
  p->n_lws = nl;
  p->n_groups = ng;
  p->n_keys = nk;
  p->m = m;
  p->max_waves = max_waves;
  p->cols = (m < max_waves ? m : max_waves) + 1u;
  return count_launch(e, lwse::launch_drain_waves(p, 0, e->sm_count, s));
}

// The buffers for n_pairs restart pairs, directly after the synchronisation that read the count.
static int reserve_drain_waves_pairs(lwse_engine* e, uint64_t n_pairs) {
  // (every index is 32-bit, and the plan kernel's items are a key's pairs times the columns)
  if (n_pairs > 0xFFFFFFFFull / (LWSE_DRAIN_WAVES_MAX + 1u)) return LWSE_ERR_OOM;
  LWSE_CUDA(e, e->dv_pairs.reserve((size_t)n_pairs * 8 + 16));
  LWSE_CUDA(e, e->dv_recs.reserve((size_t)n_pairs * 16 + 16));
  return LWSE_OK;
}

// The walk in pair mode into dv_pairs, and p's pairs set for its pass 1.
static int enqueue_drain_waves_pairs(lwse_engine* e, const lwse::DrainBudgetCostLaunch& bp, uint32_t n_pairs,
                                     lwse::DrainWavesLaunch* p) {
  LWSE_LAUNCH(e, lwse::launch_drain_restart_pairs(&bp, (unsigned long long*)e->dv_pairs.p, n_pairs, e->sm_count,
                                                  e->wf_stream));
  p->pairs = (const unsigned long long*)e->dv_pairs.p;
  p->n_pairs = n_pairs;
  p->recs = (uint4*)e->dv_recs.p;
  return LWSE_OK;
}

// The scratch of n_dense touched LWS rows, reserved, zeroed and set in p for its pass 2.
static int enqueue_drain_waves_dense(lwse_engine* e, uint32_t n_dense, lwse::DrainWavesLaunch* p) {
  cudaStream_t s = e->wf_stream;
  LWSE_CUDA(e, e->dv_lost.reserve((size_t)n_dense * p->cols * 4 + 16));
  LWSE_CUDA(e, e->dv_rwaves.reserve((size_t)n_dense * 16 + 16));
  LWSE_CUDA(e, e->dv_stamps.reserve((size_t)n_dense * 8 + 16));
  LWSE_CUDA(e, cudaMemsetAsync(e->dv_lost.p, 0, (size_t)n_dense * p->cols * 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dv_rwaves.p, 0, (size_t)n_dense * 16, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dv_stamps.p, 0, (size_t)n_dense * 8, s));
  p->n_dense = n_dense;
  p->lost = (uint32_t*)e->dv_lost.p;
  p->row_waves = (unsigned long long*)e->dv_rwaves.p;
  p->stamps = (uint32_t*)e->dv_stamps.p;
  return LWSE_OK;
}

// Three host synchronisations, each sizing what follows: the restart pairs of every key (the drain budget's pass 0
// counts them per key), then the touched LWS rows (the lost counters are sized by them, not by n_lws), then the
// answer, read back with one copy.  Everything reads the resident tables and the baseline results in place.
LWSE_API int lwse_resident_drain_waves(lwse_engine* e, lwse_drain_waves_query* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!drain_budget_ready(e)) return LWSE_ERR_NOT_READY;
  if (q->scope != LWSE_DRAIN_NODES && q->scope != LWSE_DRAIN_DOMAINS) return LWSE_ERR_INVALID_ARG;
  if (q->reserved || q->max_waves == 0 || q->max_waves > LWSE_DRAIN_WAVES_MAX || !q->waves) return LWSE_ERR_INVALID_ARG;
  if (q->n_ids && (!q->ids || !q->keys)) return LWSE_ERR_INVALID_ARG;
  const bool by_domain = q->scope == LWSE_DRAIN_DOMAINS;
  const uint32_t nk = by_domain ? e->n_domains : e->n_nodes, m = q->n_ids;
  const uint32_t nl = e->rn_lws, ng = e->rn_groups;
  if (const int rc = check_key_ids(e, q->ids, m, nk); rc != LWSE_OK) return rc;
  if (e->xch_world > 0) return LWSE_ERR_UNSUPPORTED;  // (a plan is not a sum over ranks)
  const size_t out_bytes = waves_answer_bytes<lwse_drain_wave_key, lwse_drain_wave>(m, q->max_waves);
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, e->dv_cost.reserve((size_t)nk * sizeof(lwse_drain_budget_cost) + 16));
  LWSE_CUDA(e, e->dv_words.reserve(128));
  LWSE_CUDA(e, e->wf_words.reserve(128));
  if (const int rc = reserve_drain_waves(e, m, nk, q->max_waves, out_bytes); rc != LWSE_OK) return rc;
  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* d_words = (uint32_t*)e->dv_words.p;  // [0..15] the walk's counters, [16..19] the chain's (u64)
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  LWSE_CUDA(e, cudaMemsetAsync(d_words, 0, 128, s));
  // the key rows and their restart pairs: the drain budget's pass 0
  const lwse::DrainBudgetCostLaunch bp = restart_walk(e, by_domain, (lwse_drain_budget_cost*)e->dv_cost.p, d_words);
  lwse::DrainWavesLaunch p{};
  if (const int rc = enqueue_drain_waves_setup(e, bp, q->ids, m, q->max_waves, (unsigned long long*)(d_words + 16), &p);
      rc != LWSE_OK)
    return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_words + 16, 8, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  uint64_t n_pairs = 0;
  memcpy(&n_pairs, words, 8);
  if (const int rc = reserve_drain_waves_pairs(e, n_pairs); rc != LWSE_OK) return rc;
  if (const int rc = enqueue_drain_waves_pairs(e, bp, (uint32_t)n_pairs, &p); rc != LWSE_OK) return rc;
  LWSE_LAUNCH(e, lwse::launch_drain_waves(&p, 1, e->sm_count, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_words, 64, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 16, d_words + 16, 16, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 20, p.l_first + nl, 4, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  // (the walk found another pair count, or a bucket refused a pair: no answer rather than a wrong one)
  if (ng && words[8] != n_pairs) return LWSE_ERR_OOM;
  if (words[18] || words[19]) return LWSE_ERR_OOM;
  if (const int rc = enqueue_drain_waves_dense(e, words[20], &p); rc != LWSE_OK) return rc;
  LWSE_LAUNCH(e, lwse::launch_drain_waves(&p, 2, e->sm_count, s));
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(e->dv_host.h, p.out, out_bytes, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  copy_waves_answer(e, q);
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Drain placement
// ---------------------------------------------------------------------------
// The drain placement chain, shared by lwse_resident_drain_place_cost and lwse_resident_drain_place_waves.  Its
// steps enqueue on wf_stream and never synchronize.  The caller zeroes dp_words ([0..15] the chain's counters,
// [16..31] its restart walk's) and issues every read-back.

// The largest namespace's request count: the rows of the solve's per-CTA slices.
static uint32_t largest_namespace(const lwse_engine* e) {
  const uint32_t n_ns = e->rn_namespaces;
  uint32_t max_ns = 1;
  std::vector<uint32_t> per(n_ns, 0);
  for (uint32_t r = 0; r < e->rn_reqs; r++)
    if (e->r_req_ns[r] < n_ns) max_ns = std::max(max_ns, ++per[e->r_req_ns[r]]);
  return max_ns;
}

// The chain's scratch for nk keys, before the snapshot.
static int reserve_drain_place(lwse_engine* e, uint32_t nk) {
  const uint32_t nd = e->n_domains, nr = e->rn_reqs, ng = e->rn_groups, n_ns = e->rn_namespaces;
  LWSE_CUDA(e, e->dp_cost.reserve((size_t)nk * sizeof(lwse_drain_budget_cost) + 16));
  LWSE_CUDA(e, e->dp_words.reserve(128));
  LWSE_CUDA(e, e->dp_domfree.reserve((size_t)nd * 4 + 16));
  LWSE_CUDA(e, e->dp_gidx.reserve(((size_t)ng * 3 + 2 + nr) * 4 + 16));
  LWSE_CUDA(e, e->dp_uidx.reserve(((size_t)nk * 3 + 2) * 4 + 16));
  LWSE_CUDA(e, e->dp_pos.reserve((size_t)nr * 4 + 16));
  LWSE_CUDA(e, e->dp_rows.reserve((size_t)nk * sizeof(lwse_drain_place_cost) + 16));
  LWSE_CUDA(e, e->dp_touched.reserve((size_t)n_ns + 16));
  LWSE_CUDA(e, e->dp_round.reserve(lwse::place_ns_scratch_bytes(e->n_nodes, nd, nr, n_ns)));
  if (e->node_index_stale) return reserve_node_index(e);  // (as the place what-if: a stale resident index is not read)
  return LWSE_OK;
}

// The chain's scratch and the walk's key rows zeroed, the node index, every namespace's request index, the restart
// walk's pass 0 (`bp`, into dp_cost with its counters at dp_words + 16), then the chain's pass 0 into p.
static int enqueue_drain_place_setup(lwse_engine* e, const lwse::DrainBudgetCostLaunch& bp, lwse::DrainPlaceLaunch* p) {
  const uint32_t nn = e->n_nodes, nd = e->n_domains, nr = e->rn_reqs, ng = e->rn_groups, n_ns = e->rn_namespaces;
  const uint32_t nk = bp.n_keys;
  const size_t round_bytes = lwse::place_ns_scratch_bytes(nn, nd, nr, n_ns);
  cudaStream_t s = e->wf_stream;
  LWSE_CUDA(e, cudaMemsetAsync(bp.cost, 0, (size_t)nk * sizeof(lwse_drain_budget_cost), s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dp_gidx.p, 0, (size_t)ng * 4 + 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dp_uidx.p, 0, (size_t)nk * 4 + 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dp_pos.p, 0xFF, (size_t)nr * 4 + 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dp_touched.p, 1, n_ns, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dp_round.p, 0, round_bytes, s));  // (the index counts start at zero)
  const uint32_t* dom_first = (const uint32_t*)e->dom_first.p;
  const uint32_t* node_order = (const uint32_t*)e->node_order.p;
  if (e->node_index_stale)
    if (const int rc = own_node_index(e, (const lwse_node_rec*)e->nodes.p, s, &dom_first, &node_order, nullptr); rc != LWSE_OK)
      return rc;
  LWSE_LAUNCH(e, lwse::launch_place_whatif_index((const lwse_place_req*)e->r_preq.p, nr, n_ns, (const uint8_t*)e->dp_touched.p,
                                                 nn, nd, e->dp_round.p, e->sm_count, s));
  // the restarted groups per key: the drain budget's pass 0 (key rows, the walk)
  LWSE_LAUNCH(e, lwse::launch_drain_budget_cost(&bp, 0, e->sm_count, s));
  p->nodes = (const lwse_node_rec*)e->nodes.p;
  p->occupancy = (const uint32_t*)e->r_occ.p;
  p->dom_first = dom_first;
  p->node_order = node_order;
  p->dom_free = (uint32_t*)e->dp_domfree.p;
  p->reqs = (const lwse_place_req*)e->r_preq.p;
  p->base = (const lwse_place_out*)e->r_pout.p;
  p->cost = bp.cost;
  p->n_nodes = nn;
  p->n_domains = nd;
  p->n_reqs = nr;
  p->n_namespaces = n_ns;
  p->n_groups = ng;
  p->n_keys = nk;
  p->by_domain = bp.by_domain;
  p->g_count = (uint32_t*)e->dp_gidx.p;
  p->g_first = p->g_count + ng;
  p->g_cursor = p->g_first + ng + 1;
  p->g_reqs = p->g_cursor + ng;  // (the pinned rows, at most nr)
  p->u_count = (uint32_t*)e->dp_uidx.p;
  p->u_first = p->u_count + nk;
  p->u_cursor = p->u_first + nk + 1;
  p->pos = (uint32_t*)e->dp_pos.p;
  p->rows = (lwse_drain_place_cost*)e->dp_rows.p;
  p->counts = (uint32_t*)e->dp_words.p;
  p->round = e->dp_round.p;
  p->round_bytes = round_bytes;
  return count_launch(e, lwse::launch_drain_place(p, 0, e->sm_count, s));
}

// The walk in pair mode into dp_pairs (reserved by the caller after the count's synchronisation), then the chain's
// pass 1: U_k counted and scanned.
static int enqueue_drain_place_pairs(lwse_engine* e, const lwse::DrainBudgetCostLaunch& bp, uint32_t n_pairs,
                                     lwse::DrainPlaceLaunch* p) {
  LWSE_LAUNCH(e, lwse::launch_drain_restart_pairs(&bp, (unsigned long long*)e->dp_pairs.p, n_pairs, e->sm_count, e->wf_stream));
  p->pairs = (const unsigned long long*)e->dp_pairs.p;
  p->n_pairs = n_pairs;
  return count_launch(e, lwse::launch_drain_place(p, 1, e->sm_count, e->wf_stream));
}

// The chain's pass 2 for n_unp unpinned rows and n_rule_b rule-(b) candidates, after the synchronisation that read
// them: U_k, positions, capacities and every key's alone row.  The solve's slices (results, unpinned list and marks
// per resident CTA) are sized from the largest namespace.  clamp_grid first clamps the grid to the items; the waves
// plan does not, since its p->grid also sizes the per-key namespace round of its steps.
static int enqueue_drain_place_solve(lwse_engine* e, uint32_t max_ns, uint32_t n_unp, uint32_t n_rule_b, bool clamp_grid,
                                     lwse::DrainPlaceLaunch* p) {
  const uint64_t item_cap = (uint64_t)n_unp + n_rule_b;
  if (item_cap > (1ull << 30)) return LWSE_ERR_OOM;  // (the table index is 32-bit)
  const uint64_t slots = table_slots(item_cap);
  uint64_t grid = (uint64_t)e->sm_count * 2u;
  if (clamp_grid && grid > item_cap) grid = item_cap ? item_cap : 1;
  while (grid > 1 && grid * max_ns * (sizeof(lwse_place_out) + 5) > (1ull << 30)) grid >>= 1;
  const size_t slice_out = align256((size_t)grid * max_ns * sizeof(lwse_place_out));
  const size_t slice_unp = align256((size_t)grid * max_ns * 4);
  LWSE_CUDA(e, e->dp_slices.reserve(slice_out + slice_unp + (size_t)grid * max_ns + 16));
  LWSE_CUDA(e, e->dp_items.reserve((size_t)slots * 8 + (size_t)item_cap * 8 + 16));
  LWSE_CUDA(e, e->dp_urows.reserve((size_t)n_unp * 4 + 16));
  p->u_rows = (uint32_t*)e->dp_urows.p;
  p->n_unpinned = n_unp;
  p->item_keys = (unsigned long long*)e->dp_items.p;
  p->item_mask = (uint32_t)(slots - 1);
  p->items = reinterpret_cast<uint2*>(p->item_keys + slots);
  p->item_capacity = (uint32_t)item_cap;
  LWSE_CUDA(e, cudaMemsetAsync(p->item_keys, 0xFF, (size_t)slots * 8, e->wf_stream));
  p->s_out = (lwse_place_out*)e->dp_slices.p;
  p->s_unpinned = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(e->dp_slices.p) + slice_out);
  p->s_marks = static_cast<uint8_t*>(e->dp_slices.p) + slice_out + slice_unp;
  p->slice_rows = max_ns;
  p->grid = (uint32_t)grid;
  return count_launch(e, lwse::launch_drain_place(p, 2, e->sm_count, e->wf_stream));
}

// Three host synchronisations, each sizing what follows: the restart pairs (the drain budget's pass 0 counts
// them per key), then U_k and the rule-(b) candidates, then the answer.  Everything reads the resident tables,
// the baseline group results and placement rows in place (nothing writes them while the call holds the mutex).
LWSE_API int lwse_resident_drain_place_cost(lwse_engine* e, uint32_t scope, lwse_drain_place_cost* out) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded || e->n_nodes == 0 || !e->r_groups_swept) return LWSE_ERR_NOT_READY;  // (the drain what-if's rule)
  if (!e->r_place_loaded || !e->r_place_current || e->n_domains == 0) return LWSE_ERR_NOT_READY;  // (the place what-if's)
  if (e->rn_namespaces == 0) return LWSE_ERR_NOT_READY;
  if (!out || (scope != LWSE_DRAIN_NODES && scope != LWSE_DRAIN_DOMAINS)) return LWSE_ERR_INVALID_ARG;
  if (e->xch_world > 0 || e->rn_reqs >= (1u << 24) || !lwse::place_ns_supported(e->n_nodes, e->n_domains))
    return LWSE_ERR_UNSUPPORTED;
  const bool by_domain = scope == LWSE_DRAIN_DOMAINS;
  const uint32_t nk = by_domain ? e->n_domains : e->n_nodes;
  const uint32_t max_ns = largest_namespace(e);
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, e->wf_words.reserve(256));  // (the counters, and |U| at word 32)
  if (const int rc = reserve_drain_place(e, nk); rc != LWSE_OK) return rc;
  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* d_words = (uint32_t*)e->dp_words.p;  // [0..15] this call's counters, [16..31] the walk's
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  LWSE_CUDA(e, cudaMemsetAsync(d_words, 0, 128, s));
  const lwse::DrainBudgetCostLaunch bp = restart_walk(e, by_domain, (lwse_drain_budget_cost*)e->dp_cost.p, d_words + 16);
  lwse::DrainPlaceLaunch p{};
  if (const int rc = enqueue_drain_place_setup(e, bp, &p); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_words, 32, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint32_t n_pairs = words[6];
  // the restart pairs, then U_k counted and scanned
  LWSE_CUDA(e, e->dp_pairs.reserve((size_t)n_pairs * 8 + 16));
  if (const int rc = enqueue_drain_place_pairs(e, bp, n_pairs, &p); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_words, 128, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 32, p.u_first + nk, 4, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  if (words[16 + 8] != n_pairs) return LWSE_ERR_OOM;  // (the walk found another pair count: no answer rather than a wrong one)
  if (const int rc = enqueue_drain_place_solve(e, max_ns, words[32], words[3], /*clamp_grid=*/true, &p); rc != LWSE_OK)
    return rc;
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(out, p.rows, (size_t)nk * sizeof(lwse_drain_place_cost), cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_words, 64, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  if (words[5]) return LWSE_ERR_OOM;  // an item the table refused
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Drain placement waves
// ---------------------------------------------------------------------------
// Setup: the drain waves chain up to its dense rows, then the drain placement's three passes (its per-key solve
// gives every key's alone row), then the rule-(b) domain index.  Then one captured step per key, replayed m times
// with the cursor in device memory (no host synchronisation per key), the finish, and one copy back.
LWSE_API int lwse_resident_drain_place_waves(lwse_engine* e, lwse_drain_place_waves_query* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!drain_budget_ready(e)) return LWSE_ERR_NOT_READY;
  if (!e->r_place_loaded || !e->r_place_current || e->n_domains == 0 || e->rn_namespaces == 0) return LWSE_ERR_NOT_READY;
  if (q->scope != LWSE_DRAIN_NODES && q->scope != LWSE_DRAIN_DOMAINS) return LWSE_ERR_INVALID_ARG;
  if (q->reserved || q->reserved1 || q->max_waves == 0 || q->max_waves > LWSE_DRAIN_WAVES_MAX || !q->waves) return LWSE_ERR_INVALID_ARG;
  if (q->constraints == 0 || (q->constraints & ~LWSE_DPW_ALL)) return LWSE_ERR_INVALID_ARG;
  if (q->n_ids && (!q->ids || !q->keys)) return LWSE_ERR_INVALID_ARG;
  const bool by_domain = q->scope == LWSE_DRAIN_DOMAINS;
  const uint32_t nn = e->n_nodes, nd = e->n_domains, nk = by_domain ? nd : nn, m = q->n_ids;
  const uint32_t nl = e->rn_lws, ng = e->rn_groups, nr = e->rn_reqs, n_ns = e->rn_namespaces;
  if (const int rc = check_key_ids(e, q->ids, m, nk); rc != LWSE_OK) return rc;
  if (e->xch_world > 0 || nr >= (1u << 24) || !lwse::place_ns_supported(nn, nd)) return LWSE_ERR_UNSUPPORTED;
  const uint32_t mw = q->max_waves;
  const uint32_t max_ns = largest_namespace(e);
  const size_t out_bytes = waves_answer_bytes<lwse_drain_place_wave_key, lwse_drain_place_wave>(m, mw);
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, e->dv_cost.reserve((size_t)nk * sizeof(lwse_drain_budget_cost) + 16));
  LWSE_CUDA(e, e->dv_words.reserve(128));
  LWSE_CUDA(e, e->wf_words.reserve(256));
  if (const int rc = reserve_drain_waves(e, m, nk, mw, out_bytes); rc != LWSE_OK) return rc;
  if (const int rc = reserve_drain_place(e, nk); rc != LWSE_OK) return rc;
  // this call's
  const size_t small_bytes = (size_t)LWSE_DRAIN_WAVES_MAX * 16 * 4 * 3 + (size_t)LWSE_DRAIN_WAVES_MAX * 4 + (size_t)m * 4;
  LWSE_CUDA(e, e->dq_state.reserve(sizeof(lwse::DpwState) + 16));
  LWSE_CUDA(e, e->dq_uwave.reserve((size_t)nr * 8 + 16));
  LWSE_CUDA(e, e->dq_kwave.reserve((size_t)nk * 8 + 16));
  LWSE_CUDA(e, e->dq_nswave.reserve((size_t)n_ns * 8 + 16));
  LWSE_CUDA(e, e->dq_drained.reserve((size_t)LWSE_DRAIN_WAVES_MAX * nd * 4 + 16));
  LWSE_CUDA(e, e->dq_small.reserve(small_bytes + 16));
  LWSE_CUDA(e, e->dq_colns.reserve((size_t)LWSE_DRAIN_WAVES_MAX * n_ns * 4 + 16));
  LWSE_CUDA(e, e->dq_items.reserve((size_t)LWSE_DRAIN_WAVES_MAX * n_ns * 8 + 16));
  LWSE_CUDA(e, e->dq_dix.reserve(((size_t)nd * 3 + 2 + nr) * 4 + 16));
  LWSE_CUDA(e, e->dq_out.reserve(out_bytes));
  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  // ---- the drain waves chain up to its pass 0 (lwse_resident_drain_waves) ----
  uint32_t* v_words = (uint32_t*)e->dv_words.p;
  LWSE_CUDA(e, cudaMemsetAsync(v_words, 0, 128, s));
  const lwse::DrainBudgetCostLaunch bp = restart_walk(e, by_domain, (lwse_drain_budget_cost*)e->dv_cost.p, v_words);
  lwse::DrainPlaceWavesLaunch d{};
  lwse::DrainWavesLaunch& w = d.w;
  if (const int rc = enqueue_drain_waves_setup(e, bp, q->ids, m, mw, (unsigned long long*)(v_words + 16), &w); rc != LWSE_OK)
    return rc;
  // ---- the drain placement's pass 0 (lwse_resident_drain_place_cost) ----
  uint32_t* p_words = (uint32_t*)e->dp_words.p;
  LWSE_CUDA(e, cudaMemsetAsync(p_words, 0, 128, s));
  const lwse::DrainBudgetCostLaunch pb = restart_walk(e, by_domain, (lwse_drain_budget_cost*)e->dp_cost.p, p_words + 16);
  lwse::DrainPlaceLaunch& p = d.p;
  if (const int rc = enqueue_drain_place_setup(e, pb, &p); rc != LWSE_OK) return rc;
  // first synchronisation: the pair totals of both chains (the same walk)
  LWSE_CUDA(e, cudaMemcpyAsync(words, v_words + 16, 8, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 2, p_words, 32, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  uint64_t n_pairs = 0;
  memcpy(&n_pairs, words, 8);
  const uint32_t all_pairs = words[2 + 6];
  if (const int rc = reserve_drain_waves_pairs(e, n_pairs); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, e->dp_pairs.reserve((size_t)all_pairs * 8 + 16));
  if (const int rc = enqueue_drain_waves_pairs(e, bp, (uint32_t)n_pairs, &w); rc != LWSE_OK) return rc;
  LWSE_LAUNCH(e, lwse::launch_drain_waves(&w, 1, e->sm_count, s));
  if (const int rc = enqueue_drain_place_pairs(e, pb, all_pairs, &p); rc != LWSE_OK) return rc;
  // second synchronisation: the touched rows, |U| and the rule-(b) count
  LWSE_CUDA(e, cudaMemcpyAsync(words, v_words, 64, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 16, v_words + 16, 16, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 20, w.l_first + nl, 4, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 32, p_words, 128, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 64, p.u_first + nk, 4, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  if (ng && words[8] != n_pairs) return LWSE_ERR_OOM;
  if (words[18] || words[19]) return LWSE_ERR_OOM;
  if (words[32 + 16 + 8] != all_pairs) return LWSE_ERR_OOM;
  if (const int rc = enqueue_drain_waves_dense(e, words[20], &w); rc != LWSE_OK) return rc;
  // the drain placement's pass 2: U_k, positions, capacities and every key's alone row
  if (const int rc = enqueue_drain_place_solve(e, max_ns, words[64], words[32 + 3], /*clamp_grid=*/false, &p); rc != LWSE_OK)
    return rc;
  // ---- this call's state, the domain index, the steps ----
  uint8_t* small = static_cast<uint8_t*>(e->dq_small.p);
  LWSE_CUDA(e, cudaMemsetAsync(e->dq_state.p, 0, sizeof(lwse::DpwState), s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dq_uwave.p, 0, (size_t)nr * 8, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dq_kwave.p, 0, (size_t)nk * 8, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dq_nswave.p, 0, (size_t)n_ns * 8, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dq_drained.p, 0, (size_t)LWSE_DRAIN_WAVES_MAX * nd * 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(small, 0, small_bytes, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dq_colns.p, 0, (size_t)LWSE_DRAIN_WAVES_MAX * n_ns * 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dq_dix.p, 0, (size_t)nd * 4 + 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dq_out.p, 0, out_bytes, s));
  d.st = (lwse::DpwState*)e->dq_state.p;
  d.constraints = q->constraints;
  d.max_waves = mw;
  d.u_wave = (unsigned long long*)e->dq_uwave.p;
  d.key_wave = (unsigned long long*)e->dq_kwave.p;
  d.ns_wave = (unsigned long long*)e->dq_nswave.p;
  d.drained = (uint32_t*)e->dq_drained.p;
  d.wnons = reinterpret_cast<uint32_t*>(small);
  d.wplace = d.wnons + LWSE_DRAIN_WAVES_MAX * 16;
  d.col_rows = d.wplace + LWSE_DRAIN_WAVES_MAX * 16;
  d.wbreach = d.col_rows + LWSE_DRAIN_WAVES_MAX * 16;
  d.kalone = d.wbreach + LWSE_DRAIN_WAVES_MAX;
  d.col_ns = (uint32_t*)e->dq_colns.p;
  d.items = (uint2*)e->dq_items.p;
  d.item_capacity = LWSE_DRAIN_WAVES_MAX * n_ns;
  d.dix_count = (uint32_t*)e->dq_dix.p;
  d.dix_first = d.dix_count + nd;
  d.dix_cursor = d.dix_first + nd + 1;
  d.dix_rows = d.dix_cursor + nd;
  d.out = (uint8_t*)e->dq_out.p;
  LWSE_LAUNCH(e, lwse::launch_drain_place_waves(&d, 0, e->sm_count, s));
  if (m) {
    cudaGraph_t graph = nullptr;
    GraphExec exec;
    LWSE_CUDA(e, cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int launched = lwse::launch_drain_place_waves(&d, 1, e->sm_count, s);
    const cudaError_t ce = cudaStreamEndCapture(s, &graph);
    if (launched < 0 || ce != cudaSuccess) {
      if (graph) cudaGraphDestroy(graph);
      return fail_cuda(e, launched < 0 ? (cudaError_t)-launched : ce);
    }
    cudaError_t ge = exec.ensure(graph);
    cudaGraphDestroy(graph);
    for (uint32_t i = 0; ge == cudaSuccess && i < m; i++) ge = cudaGraphLaunch(exec, s);
    if (ge != cudaSuccess) return fail_cuda(e, ge);
    e->launches += (uint64_t)launched * m;
  }
  LWSE_LAUNCH(e, lwse::launch_drain_place_waves(&d, 2, e->sm_count, s));
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(e->dv_host.h, d.out, out_bytes, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words, p_words, 64, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 16, &d.st->refused, 4, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  if (words[5] || words[16]) return LWSE_ERR_OOM;  // an item a table refused
  copy_waves_answer(e, q);
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// DS drain
// ---------------------------------------------------------------------------
static bool ds_drain_ready(const lwse_engine* e) { return drain_budget_ready(e) && e->rd_loaded; }

// drain_begin_locked, with the what-if stream also behind the DS stream (the last DS tick or load: nothing is
// in flight there while the mutex is held, but the call does not depend on that).
static int ds_drain_begin_locked(lwse_engine* e) {
  LWSE_CUDA(e, e->wf_stream.ensure(cudaStreamNonBlocking));
  LWSE_CUDA(e, e->ev_dd.ensure(cudaEventDisableTiming));
  LWSE_CUDA(e, cudaEventRecord(e->ev_dd, e->ds_stream));
  LWSE_CUDA(e, cudaStreamWaitEvent(e->wf_stream, e->ev_dd, 0));
  return drain_begin_locked(e);
}

// The resident DS tables with output set k of the DS drain's scratch (0: before, 1: after).
static lwse_ds_tables ds_drain_tables(const lwse_engine* e, int k) {
  lwse_ds_tables t{};
  t.ds = (const lwse_ds_rec*)e->rd_ds.p;
  t.n_ds = e->rdn_ds;
  t.roles = (const lwse_ds_role_rec*)e->rd_roles.p;
  t.n_roles = e->rdn_roles;
  t.revroles = (const lwse_ds_revrole_rec*)e->rd_revroles.p;
  t.n_revroles = e->rdn_revroles;
  t.ds_out = (lwse_ds_out*)e->dd_out[k].p;
  t.role_out = (lwse_ds_role_out*)e->dd_role_out[k].p;
  t.revrole_out = (lwse_ds_revrole_out*)e->dd_revrole_out[k].p;
  return t;
}

// The link table and the baseline LWS results (drain_budget_ready: they belong to the resident LWS rows).
static lwse::DsDrainLink ds_drain_link(const lwse_engine* e) {
  return lwse::DsDrainLink{(const lwse_ds_link*)e->rd_links.p, (const lwse_lws_rec*)e->r_lws.p,
                           (const lwse_lws_out*)e->r_lws_out.p, e->rn_lws};
}

static int reserve_ds_drain_outputs(lwse_engine* e, int sets) {
  for (int k = 0; k < sets; k++) {
    LWSE_CUDA(e, e->dd_out[k].reserve((size_t)e->rdn_ds * sizeof(lwse_ds_out) + 16));
    LWSE_CUDA(e, e->dd_role_out[k].reserve((size_t)e->rdn_roles * sizeof(lwse_ds_role_out) + 16));
    LWSE_CUDA(e, e->dd_revrole_out[k].reserve((size_t)e->rdn_revroles * sizeof(lwse_ds_revrole_out) + 16));
  }
  return LWSE_OK;
}

// Output set k zeroed (rows no DS's sweep writes read 0), then the linked sweep into it reading ready counts
// from `ready_from`; on wf_stream.
static int enqueue_ds_drain_sweep(lwse_engine* e, int k, const lwse_lws_out* ready_from) {
  cudaStream_t s = e->wf_stream;
  const lwse_ds_tables t = ds_drain_tables(e, k);
  LWSE_CUDA(e, cudaMemsetAsync(t.role_out, 0, (size_t)t.n_roles * sizeof(lwse_ds_role_out) + 16, s));
  LWSE_CUDA(e, cudaMemsetAsync(t.revrole_out, 0, (size_t)t.n_revroles * sizeof(lwse_ds_revrole_out) + 16, s));
  const lwse::DsDrainLink lk = ds_drain_link(e);
  return count_launch(e, lwse::launch_ds_drain_sweep(&t, &lk, ready_from, e->sm_count, s));
}

// The set form: the drain budget's mark → sweep (what-if group rows), lost[L] and the after copy of lws_out,
// the before and the after linked DS sweep, then one diff kernel over every DS.
LWSE_API int lwse_resident_ds_drain(lwse_engine* e, lwse_ds_drain_query* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!ds_drain_ready(e)) return LWSE_ERR_NOT_READY;
  if (q->scope != LWSE_DRAIN_NODES && q->scope != LWSE_DRAIN_DOMAINS) return LWSE_ERR_INVALID_ARG;
  if ((q->n_ids && !q->ids) || (q->capacity && !q->rows)) return LWSE_ERR_INVALID_ARG;
  const bool by_domain = q->scope == LWSE_DRAIN_DOMAINS;
  const uint32_t nn = e->n_nodes, nd = e->n_domains, n_keys = by_domain ? nd : nn;
  for (uint32_t i = 0; i < q->n_ids; i++)
    if (q->ids[i] >= n_keys) return LWSE_ERR_INVALID_ARG;
  const uint32_t nl = e->rn_lws, nds = e->rdn_ds;
  const uint32_t list_cap = q->capacity < nds ? q->capacity : nds;
  DeviceGuard guard(e->device);
  if (const int rc = reserve_drain_sweep(e); rc != LWSE_OK) return rc;
  if (const int rc = reserve_ds_drain_outputs(e, 2); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, e->wf_stage.reserve((size_t)n_keys));
  LWSE_CUDA(e, e->wf_words.reserve(128));
  LWSE_CUDA(e, e->dr_list.reserve(128));
  if (by_domain) LWSE_CUDA(e, e->dr_domains.reserve((size_t)nd + 16));
  LWSE_CUDA(e, e->dd_lost.reserve((size_t)nl * 4 + 16));
  LWSE_CUDA(e, e->dd_lws_after.reserve((size_t)nl * sizeof(lwse_lws_out) + 16));
  LWSE_CUDA(e, e->dd_rows.reserve((size_t)list_cap * sizeof(lwse_ds_drain) + 16));
  uint8_t* mask = static_cast<uint8_t*>(e->wf_stage.h);
  memset(mask, 0, n_keys);
  for (uint32_t i = 0; i < q->n_ids; i++) mask[q->ids[i]] = 1;
  if (const int rc = ds_drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* d_counts = (uint32_t*)e->dr_list.p;
  if (const int rc = enqueue_drain_set(e, mask, by_domain); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemsetAsync(d_counts, 0, 128, s));
  if (const int rc = enqueue_drain_sweep(e, d_counts, nullptr, nullptr, nullptr, 0); rc != LWSE_OK) return rc;
  LWSE_LAUNCH(e, lwse::launch_ds_drain_lost((const lwse_lws_rec*)e->r_lws.p, (const lwse_lws_out*)e->r_lws_out.p, nl,
                                            (const lwse_group_rec*)e->r_groups.p, (const lwse_group_out*)e->r_group_out.p,
                                            (const lwse_group_out*)e->dr_out.p, e->rn_groups, (uint32_t*)e->dd_lost.p,
                                            (lwse_lws_out*)e->dd_lws_after.p, e->sm_count, s));
  if (const int rc = enqueue_ds_drain_sweep(e, 0, (const lwse_lws_out*)e->r_lws_out.p); rc != LWSE_OK) return rc;
  if (const int rc = enqueue_ds_drain_sweep(e, 1, (const lwse_lws_out*)e->dd_lws_after.p); rc != LWSE_OK) return rc;
  const lwse_ds_tables after = ds_drain_tables(e, 1);
  const lwse::DsDrainLink lk = ds_drain_link(e);
  const lwse::DsDrainDiffHost h{(const lwse_ds_out*)e->dd_out[0].p, (const lwse_ds_role_out*)e->dd_role_out[0].p,
                                (const lwse_ds_revrole_out*)e->dd_revrole_out[0].p, (const uint32_t*)e->dd_lost.p,
                                (lwse_ds_drain*)e->dd_rows.p, list_cap, d_counts};
  LWSE_LAUNCH(e, lwse::launch_ds_drain_diff(&after, &lk, &h, e->sm_count, s));
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_counts, 128, cudaMemcpyDeviceToHost, s));
  if (q->role_out && e->rdn_roles)
    LWSE_CUDA(e, cudaMemcpyAsync(q->role_out, after.role_out, (size_t)e->rdn_roles * sizeof(lwse_ds_role_out), cudaMemcpyDeviceToHost, s));
  if (q->revrole_out && e->rdn_revroles)
    LWSE_CUDA(e, cudaMemcpyAsync(q->revrole_out, after.revrole_out, (size_t)e->rdn_revroles * sizeof(lwse_ds_revrole_out),
                                 cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint32_t n_touched = words[16];
  const uint32_t listed = n_touched < list_cap ? n_touched : list_cap;
  if (listed) {
    LWSE_CUDA(e, cudaMemcpyAsync(q->rows, e->dd_rows.p, (size_t)listed * sizeof(lwse_ds_drain), cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaStreamSynchronize(s));
  }
  q->n_touched = n_touched;
  q->n_service_lost = words[17];
  q->n_old_service_lost = words[18];
  q->n_stalled = words[19];
  q->n_changed = words[20];
  q->rows_touched = words[21];
  q->rows_zeroed = words[22];
  q->rows_linked = words[23];
  return LWSE_OK;
}

// The per-key form: the before sweep, the reverse link index's counts and scan, and the drain budget's key rows
// and pair count; one host synchronisation to size the index entries and the (LWS, key) table; the index fill,
// that table alone and the (row, key) pair count; a second synchronisation to size the (DS, key) table; then the
// insert and finish passes.
LWSE_API int lwse_resident_ds_drain_cost(lwse_engine* e, uint32_t scope, lwse_ds_drain_cost* out) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!ds_drain_ready(e)) return LWSE_ERR_NOT_READY;
  if (!out || (scope != LWSE_DRAIN_NODES && scope != LWSE_DRAIN_DOMAINS)) return LWSE_ERR_INVALID_ARG;
  const bool by_domain = scope == LWSE_DRAIN_DOMAINS;
  const uint32_t nn = e->n_nodes, n_keys = by_domain ? e->n_domains : nn, nl = e->rn_lws;
  const size_t cost_bytes = (size_t)n_keys * sizeof(lwse_ds_drain_cost);
  DeviceGuard guard(e->device);
  if (const int rc = reserve_ds_drain_outputs(e, 1); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, e->dr_bcost.reserve((size_t)n_keys * sizeof(lwse_drain_budget_cost) + 16));
  LWSE_CUDA(e, e->dr_bwords.reserve(64));
  LWSE_CUDA(e, e->wf_words.reserve(64));
  LWSE_CUDA(e, e->dd_cost.reserve(cost_bytes + 16));
  LWSE_CUDA(e, e->dd_index.reserve((size_t)(nl + 1) * 3 * 4 + 16));
  if (const int rc = ds_drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  // the before sweep (its ds_out gates the verdicts) and the reverse link index
  if (const int rc = enqueue_ds_drain_sweep(e, 0, (const lwse_lws_out*)e->r_lws_out.p); rc != LWSE_OK) return rc;
  const lwse_ds_tables t = ds_drain_tables(e, 0);
  const lwse::DsDrainLink lk = ds_drain_link(e);
  uint32_t* d_count = (uint32_t*)e->dd_index.p;
  uint32_t* d_first = d_count + (nl + 1);
  uint32_t* d_cursor = d_first + (nl + 1);
  uint32_t* d_words = (uint32_t*)e->dr_bwords.p;  // [0..1] (group, key) pairs [2] refused; [8..9] (row, key) pairs
                                                  // [10] refused; [12..13] reverse-index entries (all u64 but [2], [10])
  LWSE_CUDA(e, cudaMemsetAsync(d_words, 0, 64, s));
  LWSE_CUDA(e, cudaMemsetAsync(d_count, 0, (size_t)(nl + 1) * 4, s));
  LWSE_LAUNCH(e, lwse::launch_ds_drain_links(&t, &lk, d_count, d_cursor, nullptr, 0, (unsigned long long*)(d_words + 12),
                                             false, e->sm_count, s));
  LWSE_LAUNCH(e, lwse::launch_index_scan(d_count, d_first, d_cursor, nl, s));
  // the drain budget's (LWS, key) table: vals.y = lost(L, key)
  lwse::DrainBudgetCostLaunch p = restart_walk(e, by_domain, (lwse_drain_budget_cost*)e->dr_bcost.p, d_words);
  lwse::DsDrainCostLaunch c{};
  c.first = d_first;
  c.before = t.ds_out;
  c.cost = (lwse_ds_drain_cost*)e->dd_cost.p;
  c.counts = p.counts + 8;
  LWSE_CUDA(e, cudaMemsetAsync(p.cost, 0, (size_t)n_keys * sizeof(lwse_drain_budget_cost), s));
  LWSE_CUDA(e, cudaMemsetAsync(c.cost, 0, cost_bytes, s));
  LWSE_LAUNCH(e, lwse::launch_drain_budget_cost(&p, 0, e->sm_count, s));
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  LWSE_CUDA(e, cudaMemcpyAsync(words, p.counts, 64, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  uint64_t pairs = 0, n_entries = 0;
  memcpy(&pairs, words, 8);
  memcpy(&n_entries, words + 12, 8);
  // The index holds one entry per (DS, row that takes the LWS value): a row inside the ranges of several DS
  // counts once for each, so the entries are sized from this count, not from the revision-role table.
  // Both refusals come before the next launch: nothing is left in flight on wf_stream when the call returns.
  if (n_entries > (1ull << 30)) return LWSE_ERR_OOM;  // (the index is 32-bit)
  if (pairs > (1ull << 30)) return LWSE_ERR_OOM;      // (the table index is 32-bit)
  LWSE_CUDA(e, e->dd_entries.reserve((size_t)n_entries * sizeof(uint4) + 16));
  c.entries = (const uint4*)e->dd_entries.p;
  LWSE_LAUNCH(e, lwse::launch_ds_drain_links(&t, &lk, d_count, d_cursor, (uint4*)e->dd_entries.p, (uint32_t)n_entries, nullptr,
                                             true, e->sm_count, s));
  if (pairs) {
    const uint64_t slots = table_slots(pairs);
    LWSE_CUDA(e, e->dr_table.reserve((size_t)slots * (sizeof(unsigned long long) + sizeof(uint4))));
    p.keys = (unsigned long long*)e->dr_table.p;
    p.vals = reinterpret_cast<uint4*>(p.keys + slots);
    p.table_mask = (uint32_t)(slots - 1);
    LWSE_CUDA(e, cudaMemsetAsync(p.keys, 0xFF, (size_t)slots * sizeof(unsigned long long), s));
    LWSE_CUDA(e, cudaMemsetAsync(p.vals, 0, (size_t)slots * sizeof(uint4), s));
    LWSE_LAUNCH(e, lwse::launch_drain_budget_cost(&p, 2, e->sm_count, s));
    c.lws_keys = p.keys;
    c.lws_vals = p.vals;
    c.lws_mask = p.table_mask;
    LWSE_LAUNCH(e, lwse::launch_ds_drain_cost(&c, 0, e->sm_count, s));
    LWSE_CUDA(e, cudaMemcpyAsync(words, p.counts, 64, cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaStreamSynchronize(s));
    if (words[2]) return LWSE_ERR_OOM;  // an insert the (LWS, key) table refused
    uint64_t ds_pairs = 0;
    memcpy(&ds_pairs, words + 8, 8);
    if (ds_pairs) {
      if (ds_pairs > (1ull << 30)) return LWSE_ERR_OOM;
      uint64_t ds_slots = 256;
      while (ds_slots < 2 * ds_pairs) ds_slots <<= 1;
      LWSE_CUDA(e, e->dd_table.reserve((size_t)ds_slots * (sizeof(unsigned long long) + sizeof(uint2))));
      c.keys = (unsigned long long*)e->dd_table.p;
      c.vals = reinterpret_cast<uint2*>(c.keys + ds_slots);
      c.table_mask = (uint32_t)(ds_slots - 1);
      LWSE_CUDA(e, cudaMemsetAsync(c.keys, 0xFF, (size_t)ds_slots * sizeof(unsigned long long), s));
      LWSE_CUDA(e, cudaMemsetAsync(c.vals, 0, (size_t)ds_slots * sizeof(uint2), s));
      LWSE_LAUNCH(e, lwse::launch_ds_drain_cost(&c, 1, e->sm_count, s));
    }
  }
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  if (n_keys) LWSE_CUDA(e, cudaMemcpyAsync(out, c.cost, cost_bytes, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words, p.counts, 64, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  if (words[10]) return LWSE_ERR_OOM;  // an insert the (DS, key) table refused: no answer rather than a wrong one
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// DS drain waves
// ---------------------------------------------------------------------------
// The DS drain's before sweep, the drain waves chain with the DS caps, and the per-key forms of the drain budget
// and the DS drain (their key rows give the alone columns), sharing the drain budget's pass 0 and one (LWS, key)
// table.  Three host synchronisations, each sizing what follows: the pairs and the reverse link index entries, then
// the touched LWS rows and the (DS, key) pairs, then the answer.  Words of dv_words: [0..15] the budget walk's
// counters, [16..19] the drain waves' (u64), [20..22] the DS per-key form's, [24..25] the index entries (u64).
LWSE_API int lwse_resident_ds_drain_waves(lwse_engine* e, lwse_ds_drain_waves_query* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!ds_drain_ready(e)) return LWSE_ERR_NOT_READY;
  if (q->scope != LWSE_DRAIN_NODES && q->scope != LWSE_DRAIN_DOMAINS) return LWSE_ERR_INVALID_ARG;
  if (q->reserved || q->reserved1 || q->max_waves == 0 || q->max_waves > LWSE_DRAIN_WAVES_MAX || !q->waves)
    return LWSE_ERR_INVALID_ARG;
  if (q->constraints == 0 || (q->constraints & ~LWSE_DSW_ALL)) return LWSE_ERR_INVALID_ARG;
  if (q->n_ids && (!q->ids || !q->keys)) return LWSE_ERR_INVALID_ARG;
  const bool by_domain = q->scope == LWSE_DRAIN_DOMAINS;
  const uint32_t nk = by_domain ? e->n_domains : e->n_nodes, m = q->n_ids;
  const uint32_t nl = e->rn_lws, ng = e->rn_groups;
  if (const int rc = check_key_ids(e, q->ids, m, nk); rc != LWSE_OK) return rc;
  if (e->xch_world > 0) return LWSE_ERR_UNSUPPORTED;  // (a plan is not a sum over ranks)
  const uint32_t mw = q->max_waves;
  const size_t out_bytes = waves_answer_bytes<lwse_ds_drain_wave_key, lwse_ds_drain_wave>(m, mw);
  DeviceGuard guard(e->device);
  if (const int rc = reserve_ds_drain_outputs(e, 1); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, e->dr_bcost.reserve((size_t)nk * sizeof(lwse_drain_budget_cost) + 16));
  LWSE_CUDA(e, e->dd_cost.reserve((size_t)nk * sizeof(lwse_ds_drain_cost) + 16));
  LWSE_CUDA(e, e->dd_index.reserve((size_t)(nl + 1) * 3 * 4 + 16));
  LWSE_CUDA(e, e->dv_words.reserve(128));
  LWSE_CUDA(e, e->wf_words.reserve(192));
  if (const int rc = reserve_drain_waves(e, m, nk, mw, out_bytes); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, e->dx_caps.reserve((size_t)nl * 4 + 16));
  LWSE_CUDA(e, e->dx_out.reserve(out_bytes));
  if (const int rc = ds_drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* d_words = (uint32_t*)e->dv_words.p;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  uint32_t* d_count = (uint32_t*)e->dd_index.p;  // the reverse link index (count | first | cursor)
  uint32_t* d_first = d_count + (nl + 1);
  uint32_t* d_cursor = d_first + (nl + 1);
  LWSE_CUDA(e, cudaMemsetAsync(e->dd_cost.p, 0, (size_t)nk * sizeof(lwse_ds_drain_cost), s));
  LWSE_CUDA(e, cudaMemsetAsync(d_words, 0, 128, s));
  LWSE_CUDA(e, cudaMemsetAsync(d_count, 0, (size_t)(nl + 1) * 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dx_caps.p, 0, (size_t)nl * 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->dx_out.p, 0, out_bytes, s));
  // the before sweep (its ds_out gates the verdicts), the reverse link index's counts, the caps
  if (const int rc = enqueue_ds_drain_sweep(e, 0, (const lwse_lws_out*)e->r_lws_out.p); rc != LWSE_OK) return rc;
  lwse::DsDrainWavesLaunch d{};
  d.t = ds_drain_tables(e, 0);
  d.lk = ds_drain_link(e);
  d.caps = (uint32_t*)e->dx_caps.p;
  d.ds_cost = (const lwse_ds_drain_cost*)e->dd_cost.p;
  d.out = (uint8_t*)e->dx_out.p;
  d.max_waves = mw;
  LWSE_LAUNCH(e, lwse::launch_ds_drain_links(&d.t, &d.lk, d_count, d_cursor, nullptr, 0, (unsigned long long*)(d_words + 24),
                                             false, e->sm_count, s));
  LWSE_LAUNCH(e, lwse::launch_index_scan(d_count, d_first, d_cursor, nl, s));
  LWSE_LAUNCH(e, lwse::launch_ds_drain_waves(&d, nullptr, 0, e->sm_count, s));
  // the key rows, the member-pair count and the pair count: the drain budget's pass 0, then the key positions
  lwse::DrainBudgetCostLaunch bp = restart_walk(e, by_domain, (lwse_drain_budget_cost*)e->dr_bcost.p, d_words);
  lwse::DrainWavesLaunch p{};
  if (const int rc = enqueue_drain_waves_setup(e, bp, q->ids, m, mw, (unsigned long long*)(d_words + 16), &p); rc != LWSE_OK)
    return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_words, 128, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  uint64_t member_pairs = 0, n_pairs = 0, n_entries = 0;
  memcpy(&member_pairs, words, 8);
  memcpy(&n_pairs, words + 16, 8);
  memcpy(&n_entries, words + 24, 8);
  if (member_pairs > (1ull << 30) || n_entries > (1ull << 30)) return LWSE_ERR_OOM;
  if (const int rc = reserve_drain_waves_pairs(e, n_pairs); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, e->dd_entries.reserve((size_t)n_entries * sizeof(uint4) + 16));
  const uint64_t slots = table_slots(member_pairs);
  if (member_pairs) LWSE_CUDA(e, e->dr_table.reserve((size_t)slots * (sizeof(unsigned long long) + sizeof(uint4))));
  LWSE_LAUNCH(e, lwse::launch_ds_drain_links(&d.t, &d.lk, d_count, d_cursor, (uint4*)e->dd_entries.p, (uint32_t)n_entries, nullptr,
                                             true, e->sm_count, s));
  if (const int rc = enqueue_drain_waves_pairs(e, bp, (uint32_t)n_pairs, &p); rc != LWSE_OK) return rc;
  LWSE_LAUNCH(e, lwse::launch_drain_waves_capped(&p, d.caps, q->constraints, 1, e->sm_count, s));
  // the per-key forms: the (LWS, key) table with the budget columns, then the (row, key) pair count
  lwse::DsDrainCostLaunch c{};
  c.first = d_first;
  c.before = d.t.ds_out;
  c.cost = (lwse_ds_drain_cost*)e->dd_cost.p;
  c.counts = d_words + 20;
  c.entries = (const uint4*)e->dd_entries.p;
  if (member_pairs) {
    bp.keys = (unsigned long long*)e->dr_table.p;
    bp.vals = reinterpret_cast<uint4*>(bp.keys + slots);
    bp.table_mask = (uint32_t)(slots - 1);
    LWSE_CUDA(e, cudaMemsetAsync(bp.keys, 0xFF, (size_t)slots * sizeof(unsigned long long), s));
    LWSE_CUDA(e, cudaMemsetAsync(bp.vals, 0, (size_t)slots * sizeof(uint4), s));
    LWSE_LAUNCH(e, lwse::launch_drain_budget_cost(&bp, 1, e->sm_count, s));
    c.lws_keys = bp.keys;
    c.lws_vals = bp.vals;
    c.lws_mask = bp.table_mask;
    LWSE_LAUNCH(e, lwse::launch_ds_drain_cost(&c, 0, e->sm_count, s));
  }
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_words, 128, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 32, p.l_first + nl, 4, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  // (the walk found another pair count, or a bucket or the (LWS, key) table refused a pair: no answer rather than
  // a wrong one)
  if (ng && words[8] != n_pairs) return LWSE_ERR_OOM;
  if (words[18] || words[19] || words[2]) return LWSE_ERR_OOM;
  const uint32_t n_dense = words[32];
  uint64_t ds_pairs = 0;
  memcpy(&ds_pairs, words + 20, 8);
  if (ds_pairs) {
    if (ds_pairs > (1ull << 30)) return LWSE_ERR_OOM;
    const uint64_t ds_slots = table_slots(ds_pairs);
    LWSE_CUDA(e, e->dd_table.reserve((size_t)ds_slots * (sizeof(unsigned long long) + sizeof(uint2))));
    c.keys = (unsigned long long*)e->dd_table.p;
    c.vals = reinterpret_cast<uint2*>(c.keys + ds_slots);
    c.table_mask = (uint32_t)(ds_slots - 1);
    LWSE_CUDA(e, cudaMemsetAsync(c.keys, 0xFF, (size_t)ds_slots * sizeof(unsigned long long), s));
    LWSE_CUDA(e, cudaMemsetAsync(c.vals, 0, (size_t)ds_slots * sizeof(uint2), s));
    LWSE_LAUNCH(e, lwse::launch_ds_drain_cost(&c, 1, e->sm_count, s));
  }
  if (const int rc = enqueue_drain_waves_dense(e, n_dense, &p); rc != LWSE_OK) return rc;
  LWSE_LAUNCH(e, lwse::launch_drain_waves_capped(&p, d.caps, q->constraints, 2, e->sm_count, s));
  LWSE_LAUNCH(e, lwse::launch_ds_drain_waves(&d, &p, 1, e->sm_count, s));
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(e->dv_host.h, d.out, out_bytes, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_words + 20, 12, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  if (words[2]) return LWSE_ERR_OOM;  // an insert the (DS, key) table refused
  copy_waves_answer(e, q);
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// DisaggregatedSet sweep
// ---------------------------------------------------------------------------
static int check_ds_tables(const lwse_ds_tables* t) {
  if (!t) return LWSE_ERR_INVALID_ARG;
  if (t->n_ds && (!t->ds || !t->ds_out)) return LWSE_ERR_INVALID_ARG;
  if (t->n_roles && (!t->roles || !t->role_out)) return LWSE_ERR_INVALID_ARG;
  if (t->n_revroles && (!t->revroles || !t->revrole_out)) return LWSE_ERR_INVALID_ARG;
  if (!aligned16(t->ds) || !aligned16(t->roles) || !aligned16(t->revroles)) return LWSE_ERR_INVALID_ARG;
  return LWSE_OK;
}

LWSE_API int lwse_sweep_ds_device(lwse_engine* e, const lwse_ds_tables* t, void* stream) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  int rc = check_ds_tables(t);
  if (rc != LWSE_OK) return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  cudaStream_t s = stream ? (cudaStream_t)stream : e->stream;
  LWSE_LAUNCH(e, lwse::launch_ds_sweep(t, e->sm_count, s));
  return LWSE_OK;
}

LWSE_API int lwse_sweep_ds_host(lwse_engine* e, const lwse_ds_tables* h) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  int rc = check_ds_tables(h);
  if (rc != LWSE_OK) return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  cudaStream_t s = e->stream;
  const size_t b_ds = (size_t)h->n_ds * sizeof(lwse_ds_rec), b_ro = (size_t)h->n_roles * sizeof(lwse_ds_role_rec),
               b_rr = (size_t)h->n_revroles * sizeof(lwse_ds_revrole_rec);
  const size_t o_ds = (size_t)h->n_ds * sizeof(lwse_ds_out), o_ro = (size_t)h->n_roles * sizeof(lwse_ds_role_out),
               o_rr = (size_t)h->n_revroles * sizeof(lwse_ds_revrole_out);
  LWSE_CUDA(e, e->ds.reserve(b_ds + 16));
  LWSE_CUDA(e, e->ds_roles.reserve(b_ro + 16));
  LWSE_CUDA(e, e->ds_revroles.reserve(b_rr + 16));
  LWSE_CUDA(e, e->ds_out.reserve(o_ds + 16));
  LWSE_CUDA(e, e->ds_role_out.reserve(o_ro + 16));
  LWSE_CUDA(e, e->ds_revrole_out.reserve(o_rr + 16));
  if (b_ds) LWSE_CUDA(e, cudaMemcpyAsync(e->ds.p, h->ds, b_ds, cudaMemcpyHostToDevice, s));
  if (b_ro) LWSE_CUDA(e, cudaMemcpyAsync(e->ds_roles.p, h->roles, b_ro, cudaMemcpyHostToDevice, s));
  if (b_rr) LWSE_CUDA(e, cudaMemcpyAsync(e->ds_revroles.p, h->revroles, b_rr, cudaMemcpyHostToDevice, s));
  lwse_ds_tables d = *h;
  d.ds = (const lwse_ds_rec*)e->ds.p;
  d.roles = (const lwse_ds_role_rec*)e->ds_roles.p;
  d.revroles = (const lwse_ds_revrole_rec*)e->ds_revroles.p;
  d.ds_out = (lwse_ds_out*)e->ds_out.p;
  d.role_out = (lwse_ds_role_out*)e->ds_role_out.p;
  d.revrole_out = (lwse_ds_revrole_out*)e->ds_revrole_out.p;
  LWSE_LAUNCH(e, lwse::launch_ds_sweep(&d, e->sm_count, s));
  if (o_ds) LWSE_CUDA(e, cudaMemcpyAsync(h->ds_out, e->ds_out.p, o_ds, cudaMemcpyDeviceToHost, s));
  if (o_ro) LWSE_CUDA(e, cudaMemcpyAsync(h->role_out, e->ds_role_out.p, o_ro, cudaMemcpyDeviceToHost, s));
  if (o_rr) LWSE_CUDA(e, cudaMemcpyAsync(h->revrole_out, e->ds_revrole_out.p, o_rr, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Resident DS tables and the DS tick
// ---------------------------------------------------------------------------
// Neither call touches the LeaderWorkerSet ticks in flight: everything runs on ds_stream, and the
// only waits are on that stream (and on the DS tick's own sequence word).
LWSE_API int lwse_ds_resident_load(lwse_engine* e, const lwse_ds_tables* h) {
  if (!e || !h) return LWSE_ERR_INVALID_ARG;
  if ((h->n_ds && !h->ds) || (h->n_roles && !h->roles) || (h->n_revroles && !h->revroles)) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, e->ds_stream.ensure(cudaStreamNonBlocking));
  cudaStream_t s = e->ds_stream;
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  e->rd_loaded = false;  // (until every copy below succeeded)
  const size_t b_ds = (size_t)h->n_ds * sizeof(lwse_ds_rec), b_ro = (size_t)h->n_roles * sizeof(lwse_ds_role_rec),
               b_rr = (size_t)h->n_revroles * sizeof(lwse_ds_revrole_rec);
  const size_t o_ds = (size_t)h->n_ds * sizeof(lwse_ds_out), o_ro = (size_t)h->n_roles * sizeof(lwse_ds_role_out),
               o_rr = (size_t)h->n_revroles * sizeof(lwse_ds_revrole_out);
  LWSE_CUDA(e, e->rd_ds.reserve(b_ds + 16));
  LWSE_CUDA(e, e->rd_roles.reserve(b_ro + 16));
  LWSE_CUDA(e, e->rd_revroles.reserve(b_rr + 16));
  for (int k = 0; k < 2; k++) {
    LWSE_CUDA(e, e->rd_out[k].reserve(o_ds + 16));
    LWSE_CUDA(e, e->rd_role_out[k].reserve(o_ro + 16));
    LWSE_CUDA(e, e->rd_revrole_out[k].reserve(o_rr + 16));
  }
  LWSE_CUDA(e, e->rd_links.reserve((size_t)h->n_revroles * sizeof(lwse_ds_link) + 16));
  LWSE_CUDA(e, e->rd_marks.reserve((size_t)h->n_ds + 16));
  LWSE_CUDA(e, e->rd_ones.reserve((size_t)h->n_ds + 16));
  LWSE_CUDA(e, e->rd_counters.reserve(64));
  e->rd_off[0] = 256;                                     // [0] changed rows, [1] sequence word
  e->rd_off[1] = e->rd_off[0] + align256((size_t)h->n_ds * 4 + 16);
  e->rd_off[2] = e->rd_off[1] + align256(o_ds + 16);
  e->rd_off[3] = e->rd_off[2] + align256(o_ro + 16);
  LWSE_CUDA(e, e->rd_pin.reserve(e->rd_off[3] + align256(o_rr + 16)));
  if (b_ds) LWSE_CUDA(e, cudaMemcpyAsync(e->rd_ds.p, h->ds, b_ds, cudaMemcpyHostToDevice, s));
  if (b_ro) LWSE_CUDA(e, cudaMemcpyAsync(e->rd_roles.p, h->roles, b_ro, cudaMemcpyHostToDevice, s));
  if (b_rr) LWSE_CUDA(e, cudaMemcpyAsync(e->rd_revroles.p, h->revroles, b_rr, cudaMemcpyHostToDevice, s));
  // every link unlinked: lws_row = LWSE_NONE (all-ones rows)
  LWSE_CUDA(e, cudaMemsetAsync(e->rd_links.p, 0xFF, (size_t)h->n_revroles * sizeof(lwse_ds_link), s));
  LWSE_CUDA(e, cudaMemsetAsync(e->rd_marks.p, 0, (size_t)h->n_ds + 16, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->rd_ones.p, 1, (size_t)h->n_ds + 16, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->rd_counters.p, 0, 64, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  e->rdn_ds = h->n_ds;
  e->rdn_roles = h->n_roles;
  e->rdn_revroles = h->n_revroles;
  e->rd_parity = 0;
  e->rd_all = true;  // earlier results are forgotten: the first tick lists every DS
  e->rd_linked = false;
  e->last_ds_info = lwse_ds_tick_info{};
  e->rd_loaded = true;
  return LWSE_OK;
}

static bool ds_resident_table(const lwse_engine* e, uint32_t which, void** base, uint32_t* rows, uint32_t* row_bytes) {
  switch (which) {
    case LWSE_TABLE_DS: *base = e->rd_ds.p; *rows = e->rdn_ds; *row_bytes = sizeof(lwse_ds_rec); return true;
    case LWSE_TABLE_DS_ROLES: *base = e->rd_roles.p; *rows = e->rdn_roles; *row_bytes = sizeof(lwse_ds_role_rec); return true;
    case LWSE_TABLE_DS_REVROLES:
      *base = e->rd_revroles.p; *rows = e->rdn_revroles; *row_bytes = sizeof(lwse_ds_revrole_rec); return true;
    case LWSE_TABLE_DS_LINKS:
      *base = e->rd_links.p; *rows = e->rdn_revroles; *row_bytes = sizeof(lwse_ds_link); return true;
    default: return false;
  }
}

LWSE_API int lwse_ds_resident_tick(lwse_engine* e, const lwse_patch_seg* segs, uint32_t n_segs, lwse_ds_changes* out) {
  if (!e || !out || (n_segs && !segs) || n_segs > LWSE_TICK_MAX_SEGS) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->rd_loaded) return LWSE_ERR_NOT_READY;
  // every check before anything changes: a rejected tick leaves tables and outputs as they were
  size_t need = 0;
  for (uint32_t i = 0; i < n_segs; i++) {
    const lwse_patch_seg& g = segs[i];
    void* base;
    uint32_t rows, rb;
    if (!ds_resident_table(e, g.table, &base, &rows, &rb)) return LWSE_ERR_INVALID_ARG;
    if (g.n == 0) continue;
    if (!g.values) return LWSE_ERR_INVALID_ARG;
    if (g.flags & LWSE_PATCH_RANGE) {
      if ((uint64_t)g.first_row + g.n > rows) return LWSE_ERR_INVALID_ARG;
    } else {
      if (!g.rows) return LWSE_ERR_INVALID_ARG;
      for (uint32_t k = 0; k < g.n; k++)
        if (g.rows[k] >= rows) return LWSE_ERR_INVALID_ARG;
      need += align256((size_t)g.n * 4);
    }
    if (g.table == LWSE_TABLE_DS_LINKS) {  // reserved words must be zero
      const lwse_ds_link* v = static_cast<const lwse_ds_link*>(g.values);
      for (uint32_t k = 0; k < g.n; k++)
        if (v[k].reserved != 0) return LWSE_ERR_INVALID_ARG;
    }
    need += align256((size_t)g.n * rb);
  }
  DeviceGuard guard(e->device);
  cudaStream_t s = e->ds_stream;
  if (need > e->rd_stage.cap || need > e->rd_stage_dev.cap) {  // (the previous DS tick is complete: nothing reads them)
    LWSE_CUDA(e, e->rd_stage.reserve(need));
    LWSE_CUDA(e, e->rd_stage_dev.reserve(e->rd_stage.cap));
  }
  // stage every segment, then one H2D copy; range segments go on from the device copy, scattered
  // ones through scatter_rows_kernel, and every patched DS row is marked (the scatter copies a 1 there)
  lwse::ScatterSegHost sc[2 * LWSE_TICK_MAX_SEGS];
  int n_sc = 0;
  struct RangeCopy { void* dst; const void* src; size_t bytes; uint32_t ds_first, ds_n; } rc[LWSE_TICK_MAX_SEGS];
  int n_rc = 0;
  size_t cursor = 0;
  uint8_t* const hs = static_cast<uint8_t*>(e->rd_stage.h);
  uint8_t* const ds_dev = static_cast<uint8_t*>(e->rd_stage_dev.p);
  for (uint32_t i = 0; i < n_segs; i++) {
    const lwse_patch_seg& g = segs[i];
    if (g.n == 0) continue;
    void* base;
    uint32_t rows, rb;
    ds_resident_table(e, g.table, &base, &rows, &rb);
    const bool is_ds = g.table == LWSE_TABLE_DS;
    if (g.flags & LWSE_PATCH_RANGE) {
      memcpy(hs + cursor, g.values, (size_t)g.n * rb);
      rc[n_rc++] = RangeCopy{static_cast<uint8_t*>(base) + (size_t)g.first_row * rb, ds_dev + cursor, (size_t)g.n * rb,
                             g.first_row, is_ds ? g.n : 0u};
      cursor += align256((size_t)g.n * rb);
      continue;
    }
    memcpy(hs + cursor, g.rows, (size_t)g.n * 4);
    const uint32_t* d_rows = reinterpret_cast<const uint32_t*>(ds_dev + cursor);
    cursor += align256((size_t)g.n * 4);
    memcpy(hs + cursor, g.values, (size_t)g.n * rb);
    const void* d_vals = ds_dev + cursor;
    cursor += align256((size_t)g.n * rb);
    sc[n_sc++] = lwse::ScatterSegHost{base, rows, d_rows, d_vals, g.n, rb, false};
    if (is_ds) sc[n_sc++] = lwse::ScatterSegHost{e->rd_marks.p, rows, d_rows, e->rd_ones.p, g.n, 1u, false};
  }
  if (cursor) LWSE_CUDA(e, cudaMemcpyAsync(ds_dev, hs, cursor, cudaMemcpyHostToDevice, s));
  for (int k = 0; k < n_rc; k++) {
    LWSE_CUDA(e, cudaMemcpyAsync(rc[k].dst, rc[k].src, rc[k].bytes, cudaMemcpyDeviceToDevice, s));
    if (rc[k].ds_n) LWSE_CUDA(e, cudaMemsetAsync(static_cast<uint8_t*>(e->rd_marks.p) + rc[k].ds_first, 1, rc[k].ds_n, s));
  }
  for (int k = 0; k < n_sc; k += 8) {  // (one launch takes up to eight segments)
    LWSE_LAUNCH(e, lwse::launch_scatter(sc + k, n_sc - k < 8 ? n_sc - k : 8, nullptr, 0, s, false));
  }
  for (uint32_t i = 0; i < n_segs; i++)
    if (segs[i].table == LWSE_TABLE_DS_LINKS && segs[i].n) e->rd_linked = true;
  const uint32_t p = e->rd_parity, q = p ^ 1u;
  uint8_t* const pin_h = static_cast<uint8_t*>(e->rd_pin.h);
  uint8_t* const pin_d = static_cast<uint8_t*>(e->rd_pin.d);
  volatile uint32_t* hw = reinterpret_cast<volatile uint32_t*>(pin_h);
  uint32_t n_changed = 0;
  if (e->rdn_ds) {
    lwse_ds_tables t{};
    t.ds = (const lwse_ds_rec*)e->rd_ds.p;
    t.n_ds = e->rdn_ds;
    t.roles = (const lwse_ds_role_rec*)e->rd_roles.p;
    t.n_roles = e->rdn_roles;
    t.revroles = (const lwse_ds_revrole_rec*)e->rd_revroles.p;
    t.n_revroles = e->rdn_revroles;
    t.ds_out = (lwse_ds_out*)e->rd_out[p].p;
    t.role_out = (lwse_ds_role_out*)e->rd_role_out[p].p;
    t.revrole_out = (lwse_ds_revrole_out*)e->rd_revrole_out[p].p;
    const uint32_t seq = ++e->rd_seq == 0 ? ++e->rd_seq : e->rd_seq;  // (0 is the word's initial value)
    const bool linked = e->rd_linked;
    if (linked) {
      // The linked sweep reads r_lws / r_lws_out, which the LWS ticks write on the engine's stream: it
      // waits for everything enqueued there now (the most recently submitted LWS tick, in flight or
      // not) and nothing else — no drain, no dropped results.  The engine mutex is held until this call
      // has its results, so no later LWS tick can overwrite those rows while the DS kernel reads them.
      LWSE_CUDA(e, e->ev_ds_link.ensure(cudaEventDisableTiming));
      LWSE_CUDA(e, cudaEventRecord(e->ev_ds_link, e->stream));
      LWSE_CUDA(e, cudaStreamWaitEvent(s, e->ev_ds_link, 0));
    }
    const bool lws_results = e->r_loaded && e->r_swept;  // (after a load, r_lws_out is all-ones until a sweep)
    const lwse::DsTickHost a{(const lwse_ds_out*)e->rd_out[q].p, (const lwse_ds_role_out*)e->rd_role_out[q].p,
                             (const lwse_ds_revrole_out*)e->rd_revrole_out[q].p,
                             reinterpret_cast<lwse_ds_out*>(pin_d + e->rd_off[1]),
                             reinterpret_cast<lwse_ds_role_out*>(pin_d + e->rd_off[2]),
                             reinterpret_cast<lwse_ds_revrole_out*>(pin_d + e->rd_off[3]),
                             (uint8_t*)e->rd_marks.p, reinterpret_cast<uint32_t*>(pin_d + e->rd_off[0]),
                             (uint32_t*)e->rd_counters.p, reinterpret_cast<uint32_t*>(pin_d), seq, e->rd_all,
                             linked ? (const lwse_ds_link*)e->rd_links.p : nullptr, (const lwse_lws_rec*)e->r_lws.p,
                             (const lwse_lws_out*)e->r_lws_out.p, lws_results ? e->rn_lws : 0u};
    LWSE_LAUNCH(e, lwse::launch_ds_tick(&t, &a, e->sm_count, s));
    cudaError_t werr = cudaSuccess;
    if (!wait_word(hw + 1, seq, s, &werr)) {
      const cudaError_t a2 = cudaStreamSynchronize(s);
      return fail_cuda(e, werr != cudaSuccess ? werr : a2 != cudaSuccess ? a2 : cudaErrorUnknown);
    }
    n_changed = hw[0];
    e->rd_parity = q;
    e->rd_all = false;
    e->last_ds_info = linked ? lwse_ds_tick_info{1u, hw[2], hw[3], 0u, e->t_submitted} : lwse_ds_tick_info{};
  } else {
    if (n_sc || n_rc) LWSE_CUDA(e, cudaStreamSynchronize(s));
    e->last_ds_info = lwse_ds_tick_info{e->rd_linked ? 1u : 0u, 0u, 0u, 0u, 0u};
  }
  out->ds_rows = reinterpret_cast<const uint32_t*>(pin_h + e->rd_off[0]);
  out->n_changed = n_changed;
  out->reserved = 0;
  out->ds_out = reinterpret_cast<const lwse_ds_out*>(pin_h + e->rd_off[1]);
  out->role_out = reinterpret_cast<const lwse_ds_role_out*>(pin_h + e->rd_off[2]);
  out->revrole_out = reinterpret_cast<const lwse_ds_revrole_out*>(pin_h + e->rd_off[3]);
  return LWSE_OK;
}

LWSE_API int lwse_ds_resident_tick_info(lwse_engine* e, lwse_ds_tick_info* info) {
  if (!e || !info) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  *info = e->last_ds_info;
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// Rollout forecast
// ---------------------------------------------------------------------------
static int check_forecast_out(const lwse_ds_forecast_out* out, uint32_t n_ds, uint32_t n_roles) {
  if (!out || (n_ds && !out->ds) || (n_roles && !out->roles)) return LWSE_ERR_INVALID_ARG;
  return LWSE_OK;
}

// The forecast of the device tables `d` (sizes in d), on stream s, into the host outputs `out`.
// Everything it writes on the device is its own scratch; returns once `out` is filled.  The summary
// pass and the scan run first; the trajectory buffer is then sized by the rows that fit (not by
// step_capacity), so scratch grows only when a forecast needs more than any before it.
static int forecast_locked(lwse_engine* e, const lwse_ds_tables& d, lwse_ds_forecast_out* out, cudaStream_t s) {
  const uint32_t cap = out->steps ? out->step_capacity : 0u;
  LWSE_CUDA(e, e->fc_rows.reserve((size_t)d.n_revroles * sizeof(lwse_ds_revrole_rec) + 16));
  LWSE_CUDA(e, e->fc_ds_out.reserve((size_t)d.n_ds * sizeof(lwse_ds_out) + 16));
  LWSE_CUDA(e, e->fc_role_out.reserve((size_t)d.n_roles * sizeof(lwse_ds_role_out) + 16));
  LWSE_CUDA(e, e->fc_revrole_out.reserve((size_t)d.n_revroles * sizeof(lwse_ds_revrole_out) + 16));
  LWSE_CUDA(e, e->fc_ds.reserve((size_t)d.n_ds * sizeof(lwse_ds_forecast) + 16));
  LWSE_CUDA(e, e->fc_roles.reserve((size_t)d.n_roles * sizeof(lwse_ds_forecast_role) + 16));
  LWSE_CUDA(e, e->fc_totals.reserve(16 + (size_t)lwse::forecast_scan_words(d.n_ds) * 8));  // + the scan's block sums
  LWSE_CUDA(e, e->fc_words.reserve(16));
  const size_t b_fc = (size_t)d.n_ds * sizeof(lwse_ds_forecast), b_fr = (size_t)d.n_roles * sizeof(lwse_ds_forecast_role);
  // role rows of no valid DS read as zero
  if (b_fr) LWSE_CUDA(e, cudaMemsetAsync(e->fc_roles.p, 0, b_fr, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->fc_totals.p, 0, 16, s));
  lwse::DsForecastHost h{(lwse_ds_revrole_rec*)e->fc_rows.p, (lwse_ds_out*)e->fc_ds_out.p,
                         (lwse_ds_role_out*)e->fc_role_out.p, (lwse_ds_revrole_out*)e->fc_revrole_out.p,
                         (lwse_ds_forecast*)e->fc_ds.p, (lwse_ds_forecast_role*)e->fc_roles.p,
                         nullptr, cap, out->steps != nullptr, (unsigned long long*)e->fc_totals.p};
  LWSE_LAUNCH(e, lwse::launch_ds_forecast(&d, &h, false, e->sm_count, s));
  uint64_t* words = static_cast<uint64_t*>(e->fc_words.h);
  LWSE_CUDA(e, cudaMemcpyAsync(words, e->fc_totals.p, 16, cudaMemcpyDeviceToHost, s));
  if (b_fc) LWSE_CUDA(e, cudaMemcpyAsync(out->ds, e->fc_ds.p, b_fc, cudaMemcpyDeviceToHost, s));
  if (b_fr) LWSE_CUDA(e, cudaMemcpyAsync(out->roles, e->fc_roles.p, b_fr, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  // the DS whose rows fit come first in DS order: the written rows are [0, n_steps_written), and
  // n_steps_written <= step_capacity
  const uint32_t written = d.n_ds ? (uint32_t)words[1] : 0u;
  const uint64_t needed = d.n_ds ? words[0] : 0u;
  if (written) {
    LWSE_CUDA(e, e->fc_steps.reserve((size_t)written * sizeof(lwse_ds_role_out) + 16));
    h.steps = (lwse_ds_role_out*)e->fc_steps.p;
    LWSE_LAUNCH(e, lwse::launch_ds_forecast(&d, &h, true, e->sm_count, s));
    LWSE_CUDA(e, cudaMemcpyAsync(out->steps, e->fc_steps.p, (size_t)written * sizeof(lwse_ds_role_out),
                                 cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaStreamSynchronize(s));
  }
  out->n_steps_written = written;
  out->n_steps_needed = needed;
  return LWSE_OK;
}

LWSE_API int lwse_ds_forecast_host(lwse_engine* e, const lwse_ds_tables* h, lwse_ds_forecast_out* out) {
  if (!e || !h) return LWSE_ERR_INVALID_ARG;
  if ((h->n_ds && !h->ds) || (h->n_roles && !h->roles) || (h->n_revroles && !h->revroles)) return LWSE_ERR_INVALID_ARG;
  if (!aligned16(h->ds) || !aligned16(h->roles) || !aligned16(h->revroles)) return LWSE_ERR_INVALID_ARG;
  int rc = check_forecast_out(out, h->n_ds, h->n_roles);
  if (rc != LWSE_OK) return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  cudaStream_t s = e->stream;
  const size_t b_ds = (size_t)h->n_ds * sizeof(lwse_ds_rec), b_ro = (size_t)h->n_roles * sizeof(lwse_ds_role_rec),
               b_rr = (size_t)h->n_revroles * sizeof(lwse_ds_revrole_rec);
  LWSE_CUDA(e, e->ds.reserve(b_ds + 16));
  LWSE_CUDA(e, e->ds_roles.reserve(b_ro + 16));
  LWSE_CUDA(e, e->ds_revroles.reserve(b_rr + 16));
  if (b_ds) LWSE_CUDA(e, cudaMemcpyAsync(e->ds.p, h->ds, b_ds, cudaMemcpyHostToDevice, s));
  if (b_ro) LWSE_CUDA(e, cudaMemcpyAsync(e->ds_roles.p, h->roles, b_ro, cudaMemcpyHostToDevice, s));
  if (b_rr) LWSE_CUDA(e, cudaMemcpyAsync(e->ds_revroles.p, h->revroles, b_rr, cudaMemcpyHostToDevice, s));
  lwse_ds_tables d{};
  d.ds = (const lwse_ds_rec*)e->ds.p;
  d.n_ds = h->n_ds;
  d.roles = (const lwse_ds_role_rec*)e->ds_roles.p;
  d.n_roles = h->n_roles;
  d.revroles = (const lwse_ds_revrole_rec*)e->ds_revroles.p;
  d.n_revroles = h->n_revroles;
  return forecast_locked(e, d, out, s);
}

// On the DS stream, over rd_ds / rd_roles / rd_revroles as the last DS tick left them; the tick's
// output sets, marks, counters, pinned mirrors and links are not touched.
LWSE_API int lwse_ds_resident_forecast(lwse_engine* e, lwse_ds_forecast_out* out) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->rd_loaded) return LWSE_ERR_NOT_READY;
  int rc = check_forecast_out(out, e->rdn_ds, e->rdn_roles);
  if (rc != LWSE_OK) return rc;
  DeviceGuard guard(e->device);
  lwse_ds_tables d{};
  d.ds = (const lwse_ds_rec*)e->rd_ds.p;
  d.n_ds = e->rdn_ds;
  d.roles = (const lwse_ds_role_rec*)e->rd_roles.p;
  d.n_roles = e->rdn_roles;
  d.revroles = (const lwse_ds_revrole_rec*)e->rd_revroles.p;
  d.n_revroles = e->rdn_revroles;
  return forecast_locked(e, d, out, e->ds_stream);
}

// ---- DS rollout what-if ----
// On wf_stream behind an event on the DS stream and one on the engine's stream (ds_drain_begin_locked); reads the
// resident DS rows, link rows and LWS results in place (the mutex keeps the next tick of either kind out until the
// call returns).  The layout sizes the gathered tables at one synchronisation; the gather, the linked sweep of the
// proposed rows and the forecast over them follow.  `now` is copied out last.
LWSE_API int lwse_resident_ds_rollout_whatif(lwse_engine* e, lwse_ds_rollout_whatif* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->rd_loaded) return LWSE_ERR_NOT_READY;
  if (q->reserved) return LWSE_ERR_INVALID_ARG;
  const uint32_t n = q->n;
  if (n > LWSE_DS_WHATIF_MAX_PROPOSALS) return LWSE_ERR_UNSUPPORTED;
  if (n && (!q->proposals || !q->now || !q->fc.ds || !q->fc.roles)) return LWSE_ERR_INVALID_ARG;
  bool any_roles = false;
  for (uint32_t i = 0; i < n; i++) {
    const lwse_ds_proposal p = q->proposals[i];
    if (p.ds >= e->rdn_ds || (p.flags & ~(LWSE_DSP_NEW_REVISION | LWSE_DSP_ROLES))) return LWSE_ERR_INVALID_ARG;
    any_roles |= (p.flags & LWSE_DSP_ROLES) != 0;
  }
  if (any_roles && (!q->roles || !aligned16(q->roles))) return LWSE_ERR_INVALID_ARG;
  if (n == 0) {
    q->fc.n_steps_written = 0;
    q->fc.n_steps_needed = 0;
    return LWSE_OK;
  }
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, e->wf_stream.ensure(cudaStreamNonBlocking));
  cudaStream_t s = e->wf_stream;
  const size_t nr = (size_t)n * LWSE_DS_MAX_ROLES;
  LWSE_CUDA(e, e->dw_props.reserve((size_t)n * sizeof(lwse_ds_proposal) + 16));
  if (any_roles) LWSE_CUDA(e, e->dw_qroles.reserve(nr * sizeof(lwse_ds_role_rec) + 16));
  LWSE_CUDA(e, e->dw_count.reserve((size_t)n * 4 + 16));
  LWSE_CUDA(e, e->dw_off.reserve((size_t)n * 4 + 16));
  LWSE_CUDA(e, e->dw_sums.reserve(16 + (size_t)lwse::forecast_scan_words(n) * 8));  // [0] total, then the block sums
  LWSE_CUDA(e, e->dw_ds.reserve((size_t)n * sizeof(lwse_ds_rec) + 16));
  LWSE_CUDA(e, e->dw_roles.reserve(nr * sizeof(lwse_ds_role_rec) + 16));
  LWSE_CUDA(e, e->dw_now.reserve((size_t)n * sizeof(lwse_ds_out) + 16));
  LWSE_CUDA(e, e->dw_role_out.reserve(nr * sizeof(lwse_ds_role_out) + 16));
  LWSE_CUDA(e, e->dw_words.reserve(16));
  LWSE_CUDA(e, cudaMemcpyAsync(e->dw_props.p, q->proposals, (size_t)n * sizeof(lwse_ds_proposal), cudaMemcpyHostToDevice, s));
  if (any_roles)
    LWSE_CUDA(e, cudaMemcpyAsync(e->dw_qroles.p, q->roles, nr * sizeof(lwse_ds_role_rec), cudaMemcpyHostToDevice, s));
  if (const int rc = ds_drain_begin_locked(e); rc != LWSE_OK) return rc;
  lwse::DsWhatifHost h{};
  h.t.ds = (const lwse_ds_rec*)e->rd_ds.p;
  h.t.n_ds = e->rdn_ds;
  h.t.roles = (const lwse_ds_role_rec*)e->rd_roles.p;
  h.t.n_roles = e->rdn_roles;
  h.t.revroles = (const lwse_ds_revrole_rec*)e->rd_revroles.p;
  h.t.n_revroles = e->rdn_revroles;
  h.links = (const lwse_ds_link*)e->rd_links.p;
  h.proposals = (const lwse_ds_proposal*)e->dw_props.p;
  h.q_roles = any_roles ? (const lwse_ds_role_rec*)e->dw_qroles.p : nullptr;
  h.n = n;
  h.count = (uint32_t*)e->dw_count.p;
  h.off = (uint32_t*)e->dw_off.p;
  h.s_ds = (lwse_ds_rec*)e->dw_ds.p;
  h.s_roles = (lwse_ds_role_rec*)e->dw_roles.p;
  unsigned long long* d_sums = (unsigned long long*)e->dw_sums.p;
  LWSE_LAUNCH(e, lwse::launch_ds_whatif_layout(&h, d_sums + 2, d_sums, e->sm_count, s));
  uint64_t* words = static_cast<uint64_t*>(e->dw_words.h);
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_sums, 8, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint32_t nrr = (uint32_t)words[0];  // <= 330 n < 2^32 (the cap on n)
  LWSE_CUDA(e, e->dw_revroles.reserve((size_t)nrr * sizeof(lwse_ds_revrole_rec) + 16));
  LWSE_CUDA(e, e->dw_links.reserve((size_t)nrr * sizeof(lwse_ds_link) + 16));
  LWSE_CUDA(e, e->dw_revrole_out.reserve((size_t)nrr * sizeof(lwse_ds_revrole_out) + 16));
  h.s_revroles = (lwse_ds_revrole_rec*)e->dw_revroles.p;
  h.s_links = (lwse_ds_link*)e->dw_links.p;
  LWSE_LAUNCH(e, lwse::launch_ds_whatif_gather(&h, e->sm_count, s));
  // the DS tick's first decision over the proposed rows: the linked sweep under the tick's link state (linked only
  // after a link patch since the DS load; LWS results only while the LWS rows are loaded and swept)
  lwse_ds_tables t{};
  t.ds = (const lwse_ds_rec*)e->dw_ds.p;
  t.n_ds = n;
  t.roles = (const lwse_ds_role_rec*)e->dw_roles.p;
  t.n_roles = (uint32_t)nr;
  t.revroles = (const lwse_ds_revrole_rec*)e->dw_revroles.p;
  t.n_revroles = nrr;
  t.ds_out = (lwse_ds_out*)e->dw_now.p;
  t.role_out = (lwse_ds_role_out*)e->dw_role_out.p;
  t.revrole_out = (lwse_ds_revrole_out*)e->dw_revrole_out.p;
  LWSE_CUDA(e, cudaMemsetAsync(t.role_out, 0, nr * sizeof(lwse_ds_role_out), s));  // role rows no sweep writes read 0
  const bool lws_results = e->rd_linked && e->r_loaded && e->r_swept;
  const lwse::DsDrainLink lk{(const lwse_ds_link*)e->dw_links.p, (const lwse_lws_rec*)e->r_lws.p,
                             (const lwse_lws_out*)e->r_lws_out.p, lws_results ? e->rn_lws : 0u};
  LWSE_LAUNCH(e, lwse::launch_ds_drain_sweep(&t, &lk, lk.lws_out, e->sm_count, s));
  if (const int rc = forecast_locked(e, t, &q->fc, s); rc != LWSE_OK) return rc;
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(q->now, t.ds_out, (size_t)n * sizeof(lwse_ds_out), cudaMemcpyDeviceToHost, s));
  if (q->now_roles)
    LWSE_CUDA(e, cudaMemcpyAsync(q->now_roles, t.role_out, nr * sizeof(lwse_ds_role_out), cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  return LWSE_OK;
}

// ---- rolling-update forecast of the LeaderWorkerSets ----
// The forecast of device rows h.lws / h.group_out (sizes in h) on stream s into the host outputs `out`
// (out->lws null: the rows stay in lf_fc on the device only).
// Everything it writes on the device is its own scratch; returns once `out` is filled.  The slot layout
// comes first (it sizes the private flag bytes), then the summary pass and the scan; the trajectory
// buffer is sized by the rows that fit (not by step_capacity), so scratch only grows when a forecast
// needs more than any before it.
static int lws_forecast_locked(lwse_engine* e, lwse::LwsForecastHost& h, lwse_lws_forecast_out* out, cudaStream_t s) {
  h.step_capacity = out->steps ? out->step_capacity : 0u;
  h.want_steps = out->steps != nullptr;
  LWSE_CUDA(e, e->lf_slot_off.reserve((size_t)h.n_lws * 8 + 16));
  LWSE_CUDA(e, e->lf_fc.reserve((size_t)h.n_lws * sizeof(lwse_lws_forecast) + 16));
  LWSE_CUDA(e, e->lf_totals.reserve(32 + (size_t)lwse::forecast_scan_words(h.n_lws) * 8));  // + the scans' block sums
  LWSE_CUDA(e, e->lf_words.reserve(32));
  LWSE_CUDA(e, cudaMemsetAsync(e->lf_totals.p, 0, 32, s));
  h.slot_off = (unsigned long long*)e->lf_slot_off.p;
  h.fc = (lwse_lws_forecast*)e->lf_fc.p;
  h.totals = (unsigned long long*)e->lf_totals.p;
  uint64_t* words = static_cast<uint64_t*>(e->lf_words.h);
  LWSE_LAUNCH(e, lwse::launch_lws_forecast_slots(&h, e->sm_count, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words, e->lf_totals.p, 32, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint64_t n_slots = h.n_lws ? words[2] : 0u;
  if (n_slots >= 0x80000000ull) return LWSE_ERR_UNSUPPORTED;  // the pass indexes its slots with int32 offsets
  LWSE_CUDA(e, e->lf_slots.reserve((size_t)n_slots + 16));
  h.slots = (uint8_t*)e->lf_slots.p;
  h.n_slots = (uint32_t)n_slots;
  h.steps = nullptr;
  h.steps_rows = 0;
  LWSE_LAUNCH(e, lwse::launch_lws_forecast(&h, false, e->sm_count, s));
  const size_t b_fc = (size_t)h.n_lws * sizeof(lwse_lws_forecast);
  LWSE_CUDA(e, cudaMemcpyAsync(words, e->lf_totals.p, 32, cudaMemcpyDeviceToHost, s));
  if (b_fc && out->lws) LWSE_CUDA(e, cudaMemcpyAsync(out->lws, e->lf_fc.p, b_fc, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  // the objects whose rows fit come first in row order: the written rows are [0, n_steps_written)
  if (words[3]) return fail_cuda(e, cudaErrorAssert);  // a bounds check refused an access (an engine defect)
  const uint32_t written = h.n_lws ? (uint32_t)words[1] : 0u;
  const uint64_t needed = h.n_lws ? words[0] : 0u;
  if (written) {
    LWSE_CUDA(e, e->lf_steps.reserve((size_t)written * sizeof(lwse_lws_forecast_step) + 16));
    h.steps = (lwse_lws_forecast_step*)e->lf_steps.p;
    h.steps_rows = written;
    LWSE_LAUNCH(e, lwse::launch_lws_forecast(&h, true, e->sm_count, s));
    LWSE_CUDA(e, cudaMemcpyAsync(words, e->lf_totals.p, 32, cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaMemcpyAsync(out->steps, e->lf_steps.p, (size_t)written * sizeof(lwse_lws_forecast_step),
                                 cudaMemcpyDeviceToHost, s));
    LWSE_CUDA(e, cudaStreamSynchronize(s));
    if (words[3]) return fail_cuda(e, cudaErrorAssert);
  }
  out->n_steps_written = written;
  out->n_steps_needed = needed;
  return LWSE_OK;
}

static int lws_forecast_stream(lwse_engine* e) {
  LWSE_CUDA(e, e->lf_stream.ensure(cudaStreamNonBlocking));
  return LWSE_OK;
}

LWSE_API int lwse_lws_forecast_host(lwse_engine* e, const lwse_lws_rec* lws, uint32_t n_lws,
                                    const lwse_group_out* group_out, uint32_t n_groups, lwse_lws_forecast_out* out) {
  if (!e || !out || (n_lws && (!lws || !out->lws)) || (n_groups && !group_out)) return LWSE_ERR_INVALID_ARG;
  if (!aligned16(lws) || !aligned16(group_out)) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  int rc = lws_forecast_stream(e);
  if (rc != LWSE_OK) return rc;
  cudaStream_t s = e->lf_stream;
  const size_t b_lws = (size_t)n_lws * sizeof(lwse_lws_rec), b_go = (size_t)n_groups * sizeof(lwse_group_out);
  LWSE_CUDA(e, e->lf_lws.reserve(b_lws + 16));
  LWSE_CUDA(e, e->lf_group_out.reserve(b_go + 16));
  if (b_lws) LWSE_CUDA(e, cudaMemcpyAsync(e->lf_lws.p, lws, b_lws, cudaMemcpyHostToDevice, s));
  if (b_go) LWSE_CUDA(e, cudaMemcpyAsync(e->lf_group_out.p, group_out, b_go, cudaMemcpyHostToDevice, s));
  lwse::LwsForecastHost h{};
  h.lws = (const lwse_lws_rec*)e->lf_lws.p;
  h.n_lws = n_lws;
  h.group_out = (const lwse_group_out*)e->lf_group_out.p;
  h.n_groups = n_groups;
  return lws_forecast_locked(e, h, out, s);
}

// The resident forecast's snapshot: the resident LWS rows and group results copied on stream s into the forecast's
// own buffers, and the forecast's input over them in *h.
static int forecast_snapshot(lwse_engine* e, cudaStream_t s, lwse::LwsForecastHost* h) {
  const size_t b_lws = (size_t)e->rn_lws * sizeof(lwse_lws_rec), b_go = (size_t)e->rn_groups * sizeof(lwse_group_out);
  LWSE_CUDA(e, e->lf_lws.reserve(b_lws + 16));
  LWSE_CUDA(e, e->lf_group_out.reserve(b_go + 16));
  if (b_lws) LWSE_CUDA(e, cudaMemcpyAsync(e->lf_lws.p, e->r_lws.p, b_lws, cudaMemcpyDeviceToDevice, s));
  if (b_go) LWSE_CUDA(e, cudaMemcpyAsync(e->lf_group_out.p, e->r_group_out.p, b_go, cudaMemcpyDeviceToDevice, s));
  *h = lwse::LwsForecastHost{};
  h->lws = (const lwse_lws_rec*)e->lf_lws.p;
  h->n_lws = e->rn_lws;
  h->group_out = (const lwse_group_out*)e->lf_group_out.p;
  h->n_groups = e->rn_groups;
  return LWSE_OK;
}

// Snapshot on the engine's stream, replay on lf_stream: the ticks in flight keep running, and none of
// their buffers is written.
LWSE_API int lwse_resident_forecast(lwse_engine* e, lwse_lws_forecast_out* out) {
  if (!e) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded || !e->r_groups_swept) return LWSE_ERR_NOT_READY;
  if (!out || (e->rn_lws && !out->lws)) return LWSE_ERR_INVALID_ARG;
  DeviceGuard guard(e->device);
  int rc = lws_forecast_stream(e);
  if (rc != LWSE_OK) return rc;
  LWSE_CUDA(e, e->ev_lf.ensure(cudaEventDisableTiming));
  lwse::LwsForecastHost h{};
  if (const int src = forecast_snapshot(e, e->stream, &h); src != LWSE_OK) return src;
  LWSE_CUDA(e, cudaEventRecord(e->ev_lf, e->stream));
  LWSE_CUDA(e, cudaStreamWaitEvent(e->lf_stream, e->ev_lf, 0));
  return lws_forecast_locked(e, h, out, e->lf_stream);
}

// ---- rollout what-if ----
// The chain's first scratch for n proposals, before the snapshot.
static int reserve_rollout_whatif(lwse_engine* e, uint32_t n) {
  LWSE_CUDA(e, e->rw_rows.reserve((size_t)n * 4 + 16));
  LWSE_CUDA(e, e->rw_lws.reserve((size_t)n * sizeof(lwse_lws_rec) + 16));
  LWSE_CUDA(e, e->rw_off.reserve((size_t)n * 8 + 16));
  LWSE_CUDA(e, e->rw_sums.reserve(16 + (size_t)lwse::forecast_scan_words(n) * 8));  // [0] total, then the block sums
  LWSE_CUDA(e, e->lf_words.reserve(32));
  return LWSE_OK;
}

static int upload_rollout_proposals(lwse_engine* e, const uint32_t* rows, const lwse_lws_rec* recs, uint32_t n, cudaStream_t s) {
  LWSE_CUDA(e, cudaMemcpyAsync(e->rw_rows.p, rows, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  LWSE_CUDA(e, cudaMemcpyAsync(e->rw_lws.p, recs, (size_t)n * sizeof(lwse_lws_rec), cudaMemcpyHostToDevice, s));
  return LWSE_OK;
}

// The chain on stream s over the n uploaded proposals: the layout sizes the gathered group table at one
// synchronisation; the gather, the sweep's group pass, the restore of the foreign-owned rows and the LWS pass follow,
// then the forecast over the proposals' rows into fc (its device rows stay in lf_fc).  The `now` rows are left in
// rw_now.
static int enqueue_rollout_whatif(lwse_engine* e, uint32_t n, cudaStream_t s, lwse_lws_forecast_out* fc) {
  unsigned long long* d_sums = (unsigned long long*)e->rw_sums.p;
  lwse::RolloutWhatifHost h{};
  h.lws = (const lwse_lws_rec*)e->r_lws.p;
  h.groups = (const lwse_group_rec*)e->r_groups.p;
  h.n_groups = e->rn_groups;
  h.rows = (const uint32_t*)e->rw_rows.p;
  h.n = n;
  h.off = (unsigned long long*)e->rw_off.p;
  h.s_lws = (lwse_lws_rec*)e->rw_lws.p;
  LWSE_LAUNCH(e, lwse::launch_rollout_whatif_layout(&h, d_sums + 2, d_sums, s));
  uint64_t* words = static_cast<uint64_t*>(e->lf_words.h);
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_sums, 8, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint64_t gathered = words[0];
  if (gathered >= 0x100000000ull) return LWSE_ERR_UNSUPPORTED;  // the scratch rows are indexed with uint32
  const uint32_t ng = (uint32_t)gathered;
  const uint64_t np = e->rn_pods;
  LWSE_CUDA(e, e->rw_groups.reserve((size_t)ng * sizeof(lwse_group_rec) + 16));
  LWSE_CUDA(e, e->rw_src.reserve((size_t)ng * 4 + 16));
  LWSE_CUDA(e, e->rw_group_out.reserve((size_t)ng * sizeof(lwse_group_out) + 16));
  LWSE_CUDA(e, e->rw_now.reserve((size_t)n * sizeof(lwse_lws_out) + 16));
  LWSE_CUDA(e, e->rw_scan.reserve(lwse::lws_sweep_scratch_bytes(np, ng)));
  h.s_groups = (lwse_group_rec*)e->rw_groups.p;
  h.s_src = (uint32_t*)e->rw_src.p;
  LWSE_LAUNCH(e, lwse::launch_rollout_whatif_gather(&h, e->sm_count, s));
  // the group pass over {proposal rows, gathered groups, resident pods}, no occupancy
  lwse_lws_tables d{};
  d.lws = (const lwse_lws_rec*)e->rw_lws.p;
  d.n_lws = n;
  d.groups = (const lwse_group_rec*)e->rw_groups.p;
  d.n_groups = ng;
  d.pod_state = (const lwse_pod_state*)e->r_pst.p;
  d.pod_ident = (const lwse_pod_ident*)e->r_pid.p;
  d.n_pods = np;
  d.lws_out = (lwse_lws_out*)e->rw_now.p;
  d.group_out = (lwse_group_out*)e->rw_group_out.p;
  d.flags = e->r_sweep_flags | LWSE_SWEEP_SKIP_LWS_PASS;
  const lwse_node_rec* nodes = (const lwse_node_rec*)e->nodes.p;
  LWSE_LAUNCH(e, lwse::launch_lws_sweep(&d, nodes, e->n_nodes, e->rw_scan.p, e->sm_count, s, nullptr, nullptr,
                                        /*first_mode=*/0));
  // the rows other objects own keep the resident sweep's result, where the forecast and the LWS pass read it
  LWSE_LAUNCH(e, lwse::launch_rollout_whatif_restore(h.s_src, (const lwse_group_out*)e->r_group_out.p, d.group_out,
                                                     lwse::lws_sweep_flag_column(e->rw_scan.p, np), ng, e->sm_count, s));
  d.flags = e->r_sweep_flags | LWSE_SWEEP_SKIP_GROUP_PASS | LWSE_SWEEP_SKIP_POD_SCAN;  // the LWS pass alone
  LWSE_LAUNCH(e, lwse::launch_lws_sweep(&d, nodes, e->n_nodes, e->rw_scan.p, e->sm_count, s, nullptr, nullptr,
                                        /*first_mode=*/0));
  lwse::LwsForecastHost f{};
  f.lws = (const lwse_lws_rec*)e->rw_lws.p;
  f.n_lws = n;
  f.group_out = (const lwse_group_out*)e->rw_group_out.p;
  f.n_groups = ng;
  return lws_forecast_locked(e, f, fc, s);
}

// On lf_stream behind an event on the engine's stream; reads the resident rows, groups, pods and group
// results in place (the mutex keeps the next tick out until the call returns).  `now` is copied out last, so
// that a refused forecast writes nothing.
LWSE_API int lwse_resident_rollout_whatif(lwse_engine* e, lwse_rollout_whatif* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  if (!e->r_loaded || !e->r_groups_swept) return LWSE_ERR_NOT_READY;
  const uint32_t n = q->n;
  if (n && (!q->rows || !q->recs || !q->now || !q->fc.lws)) return LWSE_ERR_INVALID_ARG;
  if (!aligned16(q->recs)) return LWSE_ERR_INVALID_ARG;
  for (uint32_t i = 0; i < n; i++)
    if (q->rows[i] >= e->rn_lws) return LWSE_ERR_INVALID_ARG;
  if (n == 0) {
    q->fc.n_steps_written = 0;
    q->fc.n_steps_needed = 0;
    return LWSE_OK;
  }
  DeviceGuard guard(e->device);
  if (const int rc = lws_forecast_stream(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, e->ev_lf.ensure(cudaEventDisableTiming));
  cudaStream_t s = e->lf_stream;
  if (const int rc = reserve_rollout_whatif(e, n); rc != LWSE_OK) return rc;
  if (const int rc = upload_rollout_proposals(e, q->rows, q->recs, n, s); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaEventRecord(e->ev_lf, e->stream));
  LWSE_CUDA(e, cudaStreamWaitEvent(s, e->ev_lf, 0));
  if (const int rc = enqueue_rollout_whatif(e, n, s, &q->fc); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(q->now, e->rw_now.p, (size_t)n * sizeof(lwse_lws_out), cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  return LWSE_OK;
}

// ---- rollout placement ----
// The chain's first part, on wf_stream behind one event on the engine's stream: the scratch sized by n and the
// resident tables, the forecast (the resident forecast's snapshot, or the rollout what-if's chain over the
// proposals), then the count kernel, read back at one synchronisation into words[0..3] (the items, max |E_i| and
// sum |E_i|, which size the slices and decide the 24-bit refusal).  Without read_back the copy is enqueued and the
// caller synchronises, after work of its own.
static int rollout_place_count(lwse_engine* e, const uint32_t* rows, const uint32_t* ns, const lwse_lws_rec* recs, uint32_t n,
                               lwse::RolloutPlaceLaunch* p, bool read_back = true) {
  const uint32_t nn = e->n_nodes, nd = e->n_domains, nr = e->rn_reqs, n_ns = e->rn_namespaces;
  const bool proposals = recs != nullptr;
  LWSE_CUDA(e, e->wf_words.reserve(128));
  LWSE_CUDA(e, e->rp_in.reserve((size_t)n * 8 + 16));
  LWSE_CUDA(e, e->rp_rows.reserve((size_t)n * sizeof(lwse_rollout_place) + 16));
  LWSE_CUDA(e, e->rp_ent.reserve((size_t)n * 16 + 16));
  LWSE_CUDA(e, e->rp_idx.reserve(((size_t)n * 3 + 1) * 4 + 16));
  LWSE_CUDA(e, e->rp_items.reserve((size_t)n * 8 + 16));
  LWSE_CUDA(e, e->rp_words.reserve(128));
  LWSE_CUDA(e, e->rp_touched.reserve((size_t)n_ns + 16));
  LWSE_CUDA(e, e->rp_round.reserve(lwse::place_ns_scratch_bytes(nn, nd, nr, n_ns)));
  if (e->node_index_stale)
    if (const int rc = reserve_node_index(e); rc != LWSE_OK) return rc;
  if (proposals)
    if (const int rc = reserve_rollout_whatif(e, n); rc != LWSE_OK) return rc;
  if (const int rc = drain_begin_locked(e); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* d_words = (uint32_t*)e->rp_words.p;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  uint32_t* d_rows_in = (uint32_t*)e->rp_in.p;
  LWSE_CUDA(e, cudaMemcpyAsync(d_rows_in, rows, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  LWSE_CUDA(e, cudaMemcpyAsync(d_rows_in + n, ns, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  LWSE_CUDA(e, cudaMemsetAsync(d_words, 0, 128, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->rp_idx.p, 0, (size_t)n * 4, s));  // (the |E_i| counts start at zero)
  // the forecast rows F_i, on the device only (lf_fc): per entry (proposals) or per resident row
  lwse_lws_forecast_out fc{};
  if (proposals) {
    if (const int rc = upload_rollout_proposals(e, rows, recs, n, s); rc != LWSE_OK) return rc;
    if (const int rc = enqueue_rollout_whatif(e, n, s, &fc); rc != LWSE_OK) return rc;
  } else {
    lwse::LwsForecastHost h{};
    if (const int rc = forecast_snapshot(e, s, &h); rc != LWSE_OK) return rc;
    if (const int rc = lws_forecast_locked(e, h, &fc, s); rc != LWSE_OK) return rc;
  }
  *p = lwse::RolloutPlaceLaunch{};
  p->lws = (const lwse_lws_rec*)e->r_lws.p;
  p->groups = (const lwse_group_rec*)e->r_groups.p;
  p->n_groups = e->rn_groups;
  p->rows = d_rows_in;
  p->ns = d_rows_in + n;
  p->recs = proposals ? (const lwse_lws_rec*)e->rw_lws.p : nullptr;
  p->fc = (const lwse_lws_forecast*)e->lf_fc.p;
  p->fc_by_row = !proposals;
  p->n = n;
  p->rows_out = (uint32_t*)e->rp_rows.p;
  p->ent = (uint4*)e->rp_ent.p;
  p->e_count = (uint32_t*)e->rp_idx.p;
  p->e_first = p->e_count + n;
  p->e_cursor = p->e_first + n + 1;
  p->items = (uint2*)e->rp_items.p;
  p->counts = d_words;
  LWSE_LAUNCH(e, lwse::launch_rollout_place(p, 0, e->sm_count, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words, d_words, 16, cudaMemcpyDeviceToHost, s));
  if (read_back) LWSE_CUDA(e, cudaStreamSynchronize(s));
  return LWSE_OK;
}

// The chain's second part, enqueued on wf_stream after the refusals: the slices, the extra rows, the baseline's
// totals, every namespace's request index, the scan, the fill, the solve and the finish.
static int rollout_place_solve(lwse_engine* e, uint32_t n_items, uint32_t max_extra, uint64_t n_extra,
                               lwse::RolloutPlaceLaunch* p) {
  const uint32_t nn = e->n_nodes, nd = e->n_domains, nr = e->rn_reqs, n_ns = e->rn_namespaces;
  cudaStream_t s = e->wf_stream;
  // the solve's slices: the largest namespace plus the largest E_i per resident CTA
  const uint64_t slice_rows = (uint64_t)largest_namespace(e) + max_extra;
  uint64_t grid = n_items ? std::min<uint64_t>((uint64_t)e->sm_count * 2u, n_items) : 0;
  while (grid > 1 && grid * slice_rows * (sizeof(lwse_place_out) + 4) > (1ull << 30)) grid >>= 1;
  if (grid && grid * slice_rows * (sizeof(lwse_place_out) + 4) > (1ull << 31)) return LWSE_ERR_OOM;
  const size_t slice_out = align256((size_t)grid * slice_rows * sizeof(lwse_place_out));
  const size_t round_bytes = lwse::place_ns_scratch_bytes(nn, nd, nr, n_ns);
  LWSE_CUDA(e, e->rp_extra.reserve((size_t)n_extra * sizeof(lwse_place_req) + 16));
  LWSE_CUDA(e, e->rp_slices.reserve(slice_out + (size_t)grid * slice_rows * 4 + 16));
  p->extra = (lwse_place_req*)e->rp_extra.p;
  p->nodes = (const lwse_node_rec*)e->nodes.p;
  p->occupancy = (const uint32_t*)e->r_occ.p;
  p->dom_first = (const uint32_t*)e->dom_first.p;
  p->node_order = (const uint32_t*)e->node_order.p;
  p->reqs = (const lwse_place_req*)e->r_preq.p;
  p->base = (const lwse_place_out*)e->r_pout.p;
  p->n_nodes = nn;
  p->n_domains = nd;
  p->n_reqs = nr;
  p->n_namespaces = n_ns;
  p->round = e->rp_round.p;
  p->round_bytes = round_bytes;
  p->s_out = (lwse_place_out*)e->rp_slices.p;
  p->s_unpinned = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(e->rp_slices.p) + slice_out);
  p->slice_rows = (uint32_t)slice_rows;
  p->grid = (uint32_t)grid;
  // the baseline's totals (a diff of the baseline rows against themselves counts them), every namespace's index
  LWSE_LAUNCH(e, lwse::launch_place_whatif_diff(p->base, p->base, 0, nr, nullptr, nullptr, nullptr, 0, p->counts + 16,
                                                e->sm_count, s));
  if (grid) {
    LWSE_CUDA(e, cudaMemsetAsync(e->rp_touched.p, 1, n_ns, s));
    LWSE_CUDA(e, cudaMemsetAsync(e->rp_round.p, 0, round_bytes, s));  // (the index counts start at zero)
    if (e->node_index_stale)
      if (const int rc = own_node_index(e, p->nodes, s, &p->dom_first, &p->node_order, nullptr); rc != LWSE_OK) return rc;
    LWSE_LAUNCH(e, lwse::launch_place_whatif_index(p->reqs, nr, n_ns, (const uint8_t*)e->rp_touched.p, nn, nd, e->rp_round.p,
                                                   e->sm_count, s));
  }
  return count_launch(e, lwse::launch_rollout_place(p, 1, e->sm_count, s));
}

// The checks both rollout placement calls make before anything is enqueued.
static int rollout_place_check(const lwse_engine* e, const uint32_t* rows, const uint32_t* ns, const lwse_lws_rec* recs,
                               uint32_t n) {
  if (!e->r_loaded || !e->r_groups_swept) return LWSE_ERR_NOT_READY;  // (the forecast's rule)
  if (!e->r_place_loaded || !e->r_place_current || e->n_nodes == 0 || e->n_domains == 0) return LWSE_ERR_NOT_READY;
  if (n && (!rows || !ns)) return LWSE_ERR_INVALID_ARG;
  if (!aligned16(recs)) return LWSE_ERR_INVALID_ARG;
  for (uint32_t i = 0; i < n; i++)
    if (rows[i] >= e->rn_lws || ns[i] >= e->rn_namespaces) return LWSE_ERR_INVALID_ARG;
  return LWSE_OK;
}

// The forecast and the count kernel, read back at one synchronisation (max |E_i| sizes the slices and decides the
// 24-bit refusal), then the scan, the extra rows, every namespace's request index, the solve and the finish, read
// back at a second.  The rows are copied out last, so that a refused call writes nothing.
LWSE_API int lwse_resident_rollout_place(lwse_engine* e, lwse_rollout_place_query* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  const uint32_t n = q->n;
  if (const int rc = rollout_place_check(e, q->rows, q->ns, q->recs, n); rc != LWSE_OK) return rc;
  if ((n && !q->out) || (q->extra_capacity && !q->extra)) return LWSE_ERR_INVALID_ARG;
  if (e->xch_world > 0 || e->rn_reqs >= (1u << 24) || !lwse::place_ns_supported(e->n_nodes, e->n_domains))
    return LWSE_ERR_UNSUPPORTED;
  if (n == 0) {
    q->n_solved = q->n_strands = 0;
    q->n_surge = q->n_stranded = 0;
    return LWSE_OK;
  }
  const uint32_t nr = e->rn_reqs;
  DeviceGuard guard(e->device);
  lwse::RolloutPlaceLaunch p{};
  if (const int rc = rollout_place_count(e, q->rows, q->ns, q->recs, n, &p); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  const uint32_t n_items = words[0], max_extra = words[1];
  const uint64_t n_extra = (uint64_t)words[2] | (uint64_t)words[3] << 32;
  if ((uint64_t)nr + max_extra >= (1ull << 24)) return LWSE_ERR_UNSUPPORTED;  // (row keys are 24-bit)
  if (n_extra >= (1ull << 32)) return LWSE_ERR_OOM;                          // (the scan's offsets are 32-bit)
  if (const int rc = rollout_place_solve(e, n_items, max_extra, n_extra, &p); rc != LWSE_OK) return rc;
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(words, p.counts, 64, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(q->out, p.rows_out, (size_t)n * sizeof(lwse_rollout_place), cudaMemcpyDeviceToHost, s));
  if (const uint64_t listed = std::min<uint64_t>(n_extra, q->extra_capacity))
    LWSE_CUDA(e, cudaMemcpyAsync(q->extra, p.extra, (size_t)listed * sizeof(lwse_place_req), cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  q->n_solved = words[4];
  q->n_strands = words[5];
  q->n_surge = (uint64_t)words[6] | (uint64_t)words[7] << 32;
  q->n_stranded = (uint64_t)words[8] | (uint64_t)words[9] << 32;
  return LWSE_OK;
}

// ---- rollout placement waves ----
// Setup: the rollout placement's chain (its rows are the alone rows), then the key rows, the ranks and the
// per-namespace key lists, read back at a third synchronisation (R, the largest T_ns and the active namespaces
// size the lists and the slices).  Then one captured round, replayed R times with the round in device memory (no
// host synchronisation per round), the finish, and one copy back.
LWSE_API int lwse_resident_rollout_place_waves(lwse_engine* e, lwse_rollout_place_waves_query* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  const uint32_t n = q->n;
  if (const int rc = rollout_place_check(e, q->rows, q->ns, q->recs, n); rc != LWSE_OK) return rc;
  if ((n && !q->keys) || !q->waves || q->reserved) return LWSE_ERR_INVALID_ARG;
  if (q->max_waves == 0 || q->max_waves > LWSE_DRAIN_WAVES_MAX) return LWSE_ERR_INVALID_ARG;
  if (q->constraints == 0 || (q->constraints & ~LWSE_RPW_ALL)) return LWSE_ERR_INVALID_ARG;
  {
    std::vector<uint32_t> sorted(q->rows, q->rows + n);
    std::sort(sorted.begin(), sorted.end());
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) return LWSE_ERR_INVALID_ARG;
  }
  if (e->xch_world > 0 || e->rn_reqs >= (1u << 24) || !lwse::place_ns_supported(e->n_nodes, e->n_domains))
    return LWSE_ERR_UNSUPPORTED;
  if (n == 0) {
    q->n_waves = q->n_planned = q->n_triggers_alone = q->n_no_wave = q->n_not_solved = 0;
    return LWSE_OK;
  }
  const uint32_t nr = e->rn_reqs, n_ns = e->rn_namespaces, mw = q->max_waves;
  DeviceGuard guard(e->device);
  lwse::RolloutPlaceWavesLaunch w{};
  lwse::RolloutPlaceLaunch& p = w.p;
  if (const int rc = rollout_place_count(e, q->rows, q->ns, q->recs, n, &p); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  const uint32_t n_items = words[0], max_extra = words[1];
  const uint64_t n_extra = (uint64_t)words[2] | (uint64_t)words[3] << 32;
  if ((uint64_t)nr + n_extra >= (1ull << 24)) return LWSE_ERR_UNSUPPORTED;  // (a wave's rows are numbered after nr)
  if (const int rc = rollout_place_solve(e, n_items, max_extra, n_extra, &p); rc != LWSE_OK) return rc;
  // the ranks and the per-namespace key lists
  const size_t out_bytes = 32 + (size_t)n * sizeof(lwse_rollout_wave_key) + LWSE_DRAIN_WAVES_MAX * sizeof(lwse_rollout_wave);
  LWSE_CUDA(e, e->rq_state.reserve(64 + LWSE_DRAIN_WAVES_MAX * 64 + 16));
  LWSE_CUDA(e, e->rq_ns.reserve(((size_t)n_ns * 5 + 1) * 4 + 16));
  LWSE_CUDA(e, e->rq_keys.reserve((size_t)n * 4 * 3 + 16));
  LWSE_CUDA(e, e->rq_slots.reserve((size_t)n * (16 + 64 + 8 + 4 + 4 + 4 * 11) + 16));
  LWSE_CUDA(e, e->rq_out.reserve(out_bytes + 16));
  LWSE_CUDA(e, e->rq_host.reserve(out_bytes + 16));
  uint32_t* st = (uint32_t*)e->rq_state.p;
  LWSE_CUDA(e, cudaMemsetAsync(st, 0, 64 + LWSE_DRAIN_WAVES_MAX * 64, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->rq_ns.p, 0, ((size_t)n_ns * 5 + 1) * 4, s));
  LWSE_CUDA(e, cudaMemsetAsync(e->rq_out.p, 0, out_bytes, s));
  w.constraints = q->constraints;
  w.max_waves = mw;
  w.st = st;
  w.wtot = st + 16;
  w.ns_count = (uint32_t*)e->rq_ns.p;
  w.ns_first = w.ns_count + n_ns;
  w.ns_cursor = w.ns_first + n_ns + 1;
  w.ns_extra = w.ns_cursor + n_ns;
  w.ns_open = w.ns_extra + n_ns;
  w.rank = (uint32_t*)e->rq_keys.p;
  w.ns_keys = w.rank + n;
  w.act = w.ns_keys + n;
  w.out = (uint8_t*)e->rq_out.p;
  LWSE_LAUNCH(e, lwse::launch_rollout_place_waves(&w, 0, e->sm_count, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 16, st, 32, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint32_t R = words[16 + 2], max_t = words[16 + 3];
  // the slots (at most one per key), the column lists and the round's slices: the largest namespace plus its
  // largest column (T_ns) per resident CTA
  w.wc = std::min(mw, std::max(R, 1u));
  uint8_t* slots = (uint8_t*)e->rq_slots.p;
  w.desc = (uint4*)slots;
  w.res = (uint32_t*)(slots + (size_t)n * 16);
  w.items = (uint2*)(w.res + (size_t)n * 16);
  w.col_n = (uint32_t*)(w.items + n);
  w.col_rows = w.col_n + n;
  w.contrib = w.col_rows + n;
  LWSE_CUDA(e, cudaMemsetAsync(w.col_n, 0, (size_t)n * 4 * 13, s));
  LWSE_CUDA(e, e->rq_col.reserve((size_t)n * w.wc * 16 + 16));
  w.col = (uint4*)e->rq_col.p;
  const uint64_t slice_rows = (uint64_t)largest_namespace(e) + max_t;
  uint64_t grid = max_t ? std::min<uint64_t>((uint64_t)e->sm_count * 2u, n) : 0;
  while (grid > 1 && grid * slice_rows * (sizeof(lwse_place_out) + 4) > (1ull << 30)) grid >>= 1;
  if (grid && grid * slice_rows * (sizeof(lwse_place_out) + 4) > (1ull << 31)) return LWSE_ERR_OOM;
  const size_t slice_out = align256((size_t)grid * slice_rows * sizeof(lwse_place_out));
  LWSE_CUDA(e, e->rq_slices.reserve(slice_out + (size_t)grid * slice_rows * 4 + 16));
  w.s_out = (lwse_place_out*)e->rq_slices.p;
  w.s_unpinned = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(e->rq_slices.p) + slice_out);
  w.slice_rows = (uint32_t)slice_rows;
  w.grid = (uint32_t)grid;
  if (R) {
    cudaGraph_t graph = nullptr;
    GraphExec exec;
    LWSE_CUDA(e, cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int launched = lwse::launch_rollout_place_waves(&w, 1, e->sm_count, s);
    const cudaError_t ce = cudaStreamEndCapture(s, &graph);
    if (launched < 0 || ce != cudaSuccess) {
      if (graph) cudaGraphDestroy(graph);
      return fail_cuda(e, launched < 0 ? (cudaError_t)-launched : ce);
    }
    cudaError_t ge = exec.ensure(graph);
    cudaGraphDestroy(graph);
    for (uint32_t r = 0; ge == cudaSuccess && r < R; r++) ge = cudaGraphLaunch(exec, s);
    if (ge != cudaSuccess) return fail_cuda(e, ge);
    e->launches += (uint64_t)launched * R;
  }
  LWSE_LAUNCH(e, lwse::launch_rollout_place_waves(&w, 2, e->sm_count, s));
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(e->rq_host.h, w.out, out_bytes, cudaMemcpyDeviceToHost, s));
  if (q->alone_rows)
    LWSE_CUDA(e, cudaMemcpyAsync(q->alone_rows, p.rows_out, (size_t)n * sizeof(lwse_rollout_place), cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint8_t* h = static_cast<const uint8_t*>(e->rq_host.h);
  uint32_t tot[5];
  memcpy(tot, h, sizeof(tot));
  memcpy(q->keys, h + 32, (size_t)n * sizeof(lwse_rollout_wave_key));
  memcpy(q->waves, h + 32 + (size_t)n * sizeof(lwse_rollout_wave_key), (size_t)tot[0] * sizeof(lwse_rollout_wave));
  q->n_waves = tot[0];
  q->n_planned = tot[1];
  q->n_triggers_alone = tot[2];
  q->n_no_wave = tot[3];
  q->n_not_solved = tot[4];
  return LWSE_OK;
}

// ---- scale headroom ----
// Setup: the rollout placement's count on the resident rows and the setup kernel, read back at one synchronisation
// (the entries that search, the largest |E| and the per-round sum of |E| size the slices, the grid and the extra
// rows; the probe at r0 would size none for a settled object with all its pods), then the rollout placement's
// solve, whose rows are the probes at r0 (the current rows), copied aside.  Then one captured round, replayed with
// the bounds in device memory (no host synchronisation per round), the finish, and one copy back.
LWSE_API int lwse_resident_scale_headroom(lwse_engine* e, lwse_scale_headroom_query* q) {
  if (!e || !q) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  const uint32_t n = q->n;
  if (const int rc = rollout_place_check(e, q->rows, q->ns, nullptr, n); rc != LWSE_OK) return rc;
  if ((n && !q->out) || q->reserved || q->reserved1) return LWSE_ERR_INVALID_ARG;
  if (!(q->constraints & LWSE_RPW_STRANDED) || (q->constraints & ~LWSE_RPW_ALL)) return LWSE_ERR_INVALID_ARG;
  if (e->xch_world > 0 || e->rn_reqs >= (1u << 24) || !lwse::place_ns_supported(e->n_nodes, e->n_domains))
    return LWSE_ERR_UNSUPPORTED;
  if (n == 0) {
    q->n_solved = q->n_blocked = q->n_at_ceiling = q->rounds = 0;
    q->headroom = 0;
    return LWSE_OK;
  }
  const uint32_t nr = e->rn_reqs;
  const size_t row_bytes = (size_t)n * 64, out_bytes = 32 + row_bytes;
  DeviceGuard guard(e->device);
  LWSE_CUDA(e, e->sh_ceil.reserve((size_t)n * 4 + 16));
  LWSE_CUDA(e, e->sh_state.reserve((size_t)n * 16 + 16));
  LWSE_CUDA(e, e->sh_rows.reserve(row_bytes * 3 + 16));
  LWSE_CUDA(e, e->sh_out.reserve(out_bytes + 32 + 16));
  LWSE_CUDA(e, e->sh_host.reserve(out_bytes + 16));
  lwse::ScaleHeadroomLaunch h{};
  lwse::RolloutPlaceLaunch& p = h.p;
  if (const int rc = rollout_place_count(e, q->rows, q->ns, nullptr, n, &p, /*read_back=*/false); rc != LWSE_OK) return rc;
  cudaStream_t s = e->wf_stream;
  uint32_t* words = static_cast<uint32_t*>(e->wf_words.h);
  h.constraints = q->constraints;
  h.n_domains = e->n_domains;
  h.st = (uint4*)e->sh_state.p;
  h.cur = (const uint32_t*)e->sh_rows.p;
  h.clean = (uint32_t*)e->sh_rows.p + (size_t)n * 16;
  h.trig = h.clean + (size_t)n * 16;
  h.out = (uint32_t*)e->sh_out.p;
  h.words = h.out + out_bytes / 4;
  if (q->ceilings) {
    LWSE_CUDA(e, cudaMemcpyAsync(e->sh_ceil.p, q->ceilings, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    h.ceilings = (const int32_t*)e->sh_ceil.p;
  }
  LWSE_CUDA(e, cudaMemsetAsync(h.out, 0, out_bytes + 32, s));
  LWSE_LAUNCH(e, lwse::launch_scale_headroom(&h, 0, e->sm_count, s));
  LWSE_CUDA(e, cudaMemcpyAsync(words + 16, h.words, 32, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  // the r0 probes (every SOLVED entry of the rollout placement) and the rounds' probes share the sizes
  const uint32_t n_items = std::max(words[0], words[16]), max_extra = std::max(words[1], words[17]);
  const uint64_t n_extra = std::max((uint64_t)words[2] | (uint64_t)words[3] << 32, (uint64_t)words[18] | (uint64_t)words[19] << 32);
  const uint32_t rounds = words[20];
  if ((uint64_t)nr + max_extra >= (1ull << 24)) return LWSE_ERR_UNSUPPORTED;  // (row keys are 24-bit)
  if (n_extra >= (1ull << 32)) return LWSE_ERR_OOM;                          // (the scan's offsets are 32-bit)
  if (const int rc = rollout_place_solve(e, n_items, max_extra, n_extra, &p); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(e->sh_rows.p, p.rows_out, row_bytes, cudaMemcpyDeviceToDevice, s));
  LWSE_CUDA(e, cudaMemsetAsync(p.counts, 0, 4, s));  // (the rounds gather their own items)
  if (rounds) {
    cudaGraph_t graph = nullptr;
    GraphExec exec;
    LWSE_CUDA(e, cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int launched = lwse::launch_scale_headroom(&h, 1, e->sm_count, s);
    const cudaError_t ce = cudaStreamEndCapture(s, &graph);
    if (launched < 0 || ce != cudaSuccess) {
      if (graph) cudaGraphDestroy(graph);
      return fail_cuda(e, launched < 0 ? (cudaError_t)-launched : ce);
    }
    cudaError_t ge = exec.ensure(graph);
    cudaGraphDestroy(graph);
    for (uint32_t r = 0; ge == cudaSuccess && r < rounds; r++) ge = cudaGraphLaunch(exec, s);
    if (ge != cudaSuccess) return fail_cuda(e, ge);
    e->launches += (uint64_t)launched * rounds;
  }
  LWSE_LAUNCH(e, lwse::launch_scale_headroom(&h, 2, e->sm_count, s));
  if (const int rc = drain_end_locked(e); rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(e->sh_host.h, h.out, out_bytes, cudaMemcpyDeviceToHost, s));
  if (q->current) LWSE_CUDA(e, cudaMemcpyAsync(q->current, h.cur, row_bytes, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  const uint8_t* hb = static_cast<const uint8_t*>(e->sh_host.h);
  uint32_t tot[6];
  memcpy(tot, hb, sizeof(tot));
  memcpy(q->out, hb + 32, row_bytes);
  q->n_solved = tot[0];
  q->n_blocked = tot[1];
  q->n_at_ceiling = tot[2];
  q->rounds = rounds;
  q->headroom = (uint64_t)tot[4] | (uint64_t)tot[5] << 32;
  return LWSE_OK;
}

// ---------------------------------------------------------------------------
// SHA-1 group keys
// ---------------------------------------------------------------------------
static int group_keys_locked(lwse_engine* e, const uint8_t* d_bytes, const uint32_t* d_offsets, uint32_t n,
                             uint8_t* d_digests, cudaStream_t s) {
  LWSE_LAUNCH(e, lwse::launch_sha1(d_bytes, d_offsets, n, d_digests, e->sm_count, s));
  return LWSE_OK;
}

LWSE_API int lwse_group_keys_device(lwse_engine* e, const uint8_t* d_bytes, const uint32_t* d_offsets,
                                    uint32_t n, uint8_t* d_digests, void* stream) {
  if (!e || (n && (!d_offsets || !d_digests))) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  return group_keys_locked(e, d_bytes, d_offsets, n, d_digests, stream ? (cudaStream_t)stream : e->stream);
}

LWSE_API int lwse_group_keys_host(lwse_engine* e, const uint8_t* bytes, const uint32_t* offsets,
                                  uint32_t n, uint8_t* digests) {
  if (!e || (n && (!offsets || !digests))) return LWSE_ERR_INVALID_ARG;
  if (n == 0) return LWSE_OK;
  const size_t total = offsets[n];
  if (total && !bytes) return LWSE_ERR_INVALID_ARG;
  // one lock for staging, launch and download (concurrent webhook admissions share the buffers)
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  cudaStream_t s = e->stream;
  LWSE_CUDA(e, e->sha_bytes.reserve(total + 64));
  LWSE_CUDA(e, e->sha_offsets.reserve((size_t)(n + 1) * 4 + 16));
  LWSE_CUDA(e, e->sha_digests.reserve((size_t)n * 20 + 16));
  if (total) LWSE_CUDA(e, cudaMemcpyAsync(e->sha_bytes.p, bytes, total, cudaMemcpyHostToDevice, s));
  LWSE_CUDA(e, cudaMemcpyAsync(e->sha_offsets.p, offsets, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, s));
  const int rc = group_keys_locked(e, (const uint8_t*)e->sha_bytes.p, (const uint32_t*)e->sha_offsets.p, n,
                                   (uint8_t*)e->sha_digests.p, s);
  if (rc != LWSE_OK) return rc;
  LWSE_CUDA(e, cudaMemcpyAsync(digests, e->sha_digests.p, (size_t)n * 20, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  return LWSE_OK;
}

LWSE_API int lwse_subgroup_keys_device(lwse_engine* e, const uint8_t* d_bytes, const uint32_t* d_offsets, uint32_t n,
                                       const int32_t* d_pod_count, const int32_t* d_subgroup_size,
                                       const int32_t* d_worker_index, int32_t* d_index_out, uint8_t* d_digests,
                                       void* stream) {
  if (!e || (n && (!d_offsets || !d_digests || !d_pod_count || !d_subgroup_size || !d_worker_index || !d_index_out)))
    return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  LWSE_LAUNCH(e, lwse::launch_subgroup_keys(d_bytes, d_offsets, n, d_pod_count, d_subgroup_size, d_worker_index, d_index_out,
                                            d_digests, e->sm_count, stream ? (cudaStream_t)stream : e->stream));
  return LWSE_OK;
}

LWSE_API int lwse_subgroup_keys_host(lwse_engine* e, const uint8_t* bytes, const uint32_t* offsets, uint32_t n,
                                     const int32_t* pod_count, const int32_t* subgroup_size,
                                     const int32_t* worker_index, int32_t* index_out, uint8_t* digests) {
  if (!e || (n && (!offsets || !digests || !pod_count || !subgroup_size || !worker_index || !index_out)))
    return LWSE_ERR_INVALID_ARG;
  if (n == 0) return LWSE_OK;
  const size_t total = offsets[n];
  if (total && !bytes) return LWSE_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> lock(e->mu);
  DeviceGuard guard(e->device);
  cudaStream_t s = e->stream;
  const size_t b_int = (size_t)n * 4;
  LWSE_CUDA(e, e->sha_bytes.reserve(total + 64));
  LWSE_CUDA(e, e->sha_offsets.reserve((size_t)(n + 1) * 4 + 16));
  LWSE_CUDA(e, e->sha_digests.reserve((size_t)n * 20 + 16));
  LWSE_CUDA(e, e->sha_ints.reserve(4 * b_int + 64));
  int32_t* d_int = static_cast<int32_t*>(e->sha_ints.p);
  if (total) LWSE_CUDA(e, cudaMemcpyAsync(e->sha_bytes.p, bytes, total, cudaMemcpyHostToDevice, s));
  LWSE_CUDA(e, cudaMemcpyAsync(e->sha_offsets.p, offsets, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, s));
  LWSE_CUDA(e, cudaMemcpyAsync(d_int, pod_count, b_int, cudaMemcpyHostToDevice, s));
  LWSE_CUDA(e, cudaMemcpyAsync(d_int + n, subgroup_size, b_int, cudaMemcpyHostToDevice, s));
  LWSE_CUDA(e, cudaMemcpyAsync(d_int + 2 * (size_t)n, worker_index, b_int, cudaMemcpyHostToDevice, s));
  LWSE_LAUNCH(e, lwse::launch_subgroup_keys((const uint8_t*)e->sha_bytes.p, (const uint32_t*)e->sha_offsets.p, n, d_int, d_int + n,
                                            d_int + 2 * (size_t)n, d_int + 3 * (size_t)n, (uint8_t*)e->sha_digests.p,
                                            e->sm_count, s));
  LWSE_CUDA(e, cudaMemcpyAsync(index_out, d_int + 3 * (size_t)n, b_int, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaMemcpyAsync(digests, e->sha_digests.p, (size_t)n * 20, cudaMemcpyDeviceToHost, s));
  LWSE_CUDA(e, cudaStreamSynchronize(s));
  return LWSE_OK;
}

}  // extern "C"
