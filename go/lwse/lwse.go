// Package lwse is the cgo binding of liblwse.so (include/lwse.h): the H100
// reconcile-and-placement engine behind the LeaderWorkerSet / DisaggregatedSet
// reconcilers.
//
// A SKETCH, NOT A BUILD ARTEFACT: this repository's image has no Go toolchain, so these two
// files (lwse.go, arena.go) have never been compiled.  They show the binding a maintainer adds
// to sigs.k8s.io/lws, kept next to the header it binds; what IS built and run here is the same
// calling pattern in C — C-malloc'd tables, several threads on one handle, the resident tick fed
// from the pinned arena — tests/host_c/cgo_pattern_check.c, driven by tests/test_cgo_pattern.py.
// Every exported function maps 1:1 to a C symbol; tables are passed as C-allocated
// (or pinned) memory because cgo forbids the C side to retain Go pointers.
package lwse

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../lws_b200 -llwse -Wl,-rpath,${SRCDIR}/../../lws_b200
#include <stdlib.h>
#include "lwse.h"
*/
import "C"

import (
	"fmt"
	"unsafe"
)

// Engine is one GPU's engine handle (lwse_create). One per device; a handle runs one
// sweep at a time.
type Engine struct{ h *C.lwse_engine }

// Error wraps a negative lwse_status.
type Error struct {
	Status int
	Cuda   int
}

func (e *Error) Error() string {
	return fmt.Sprintf("lwse: %s (status %d, cudaError %d)", C.GoString(C.lwse_strerror(C.int(e.Status))), e.Status, e.Cuda)
}

func (e *Engine) check(rc C.int) error {
	if rc == C.LWSE_OK {
		return nil
	}
	return &Error{Status: int(rc), Cuda: int(C.lwse_last_cuda_error(e.h))}
}

// New creates an engine on a CUDA device. There is no CPU fallback: without a usable
// sm_90 device this fails with LWSE_ERR_NO_DEVICE and the operator keeps its stock path.
func New(device int) (*Engine, error) {
	cfg := C.lwse_config{abi_version: C.LWSE_ABI_VERSION, device: C.int32_t(device)}
	var h *C.lwse_engine
	if rc := C.lwse_create(&cfg, &h); rc != C.LWSE_OK {
		return nil, &Error{Status: int(rc)}
	}
	return &Engine{h: h}, nil
}

func (e *Engine) Close() { C.lwse_destroy(e.h); e.h = nil }

// ShardOf: which of n engines owns an object (hash(LWS.UID) mod nGPU; DS-owned LWS pass
// the DS uid hash so a DS and its children co-reside).
func ShardOf(uidHash uint64, n uint32) uint32 { return uint32(C.lwse_shard_of(C.uint64_t(uidHash), C.uint32_t(n))) }

// Hash64 is the string hash of the encoders (revision keys, label values, UIDs).
func Hash64(s string) uint64 {
	if len(s) == 0 {
		return uint64(C.lwse_hash64(nil, 0))
	}
	b := []byte(s)
	return uint64(C.lwse_hash64(unsafe.Pointer(&b[0]), C.size_t(len(b))))
}

// Tables is a set of C-allocated record tables (see Arena in arena.go).
type LwsTables struct {
	Lws      *C.lwse_lws_rec
	NLws     uint32
	Groups   *C.lwse_group_rec
	NGroups  uint32
	PodState *C.lwse_pod_state
	PodIdent *C.lwse_pod_ident
	NPods    uint64
	LwsOut   *C.lwse_lws_out
	GroupOut *C.lwse_group_out
	Occ      *C.uint32_t // optional
	Flags    uint32
}

func (t *LwsTables) c() C.lwse_lws_tables {
	return C.lwse_lws_tables{
		lws: t.Lws, n_lws: C.uint32_t(t.NLws), groups: t.Groups, n_groups: C.uint32_t(t.NGroups),
		pod_state: t.PodState, pod_ident: t.PodIdent, n_pods: C.uint64_t(t.NPods),
		lws_out: t.LwsOut, group_out: t.GroupOut, node_occupancy: t.Occ, flags: C.uint32_t(t.Flags),
	}
}

// UploadNodes makes the node table resident (call on Node add/update/delete batches).
func (e *Engine) UploadNodes(nodes *C.lwse_node_rec, n, nDomains uint32) error {
	return e.check(C.lwse_upload_nodes(e.h, nodes, C.uint32_t(n), C.uint32_t(nDomains)))
}

// SweepLws: host tables in, host result tables out (H2D, two or three kernels, D2H, sync).  With
// pinned, mapped tables the 16-byte pod identity column is not uploaded: a prefetch kernel copies
// just the rows of pods with a restart / deletion event while the other tables cross PCIe.
func (e *Engine) SweepLws(t *LwsTables) error {
	ct := t.c()
	return e.check(C.lwse_sweep_lws_host(e.h, &ct))
}

// Place runs one placement round over host request rows.
func (e *Engine) Place(reqs *C.lwse_place_req, n uint32, occupancy *C.uint32_t, nNamespaces uint32, out *C.lwse_place_out) (rounds uint32, err error) {
	var r C.uint32_t
	err = e.check(C.lwse_place_host(e.h, reqs, C.uint32_t(n), occupancy, C.uint32_t(nNamespaces), out, &r))
	return uint32(r), err
}

// SweepDs advances every DisaggregatedSet by one reconcile.
func (e *Engine) SweepDs(t *C.lwse_ds_tables) error { return e.check(C.lwse_sweep_ds_host(e.h, t)) }

// DsResidentLoad makes the three DS input tables resident (spare rows included; the next DsTick
// lists every DS).  It never waits for the LeaderWorkerSet ticks in flight.
func (e *Engine) DsResidentLoad(t *C.lwse_ds_tables) error { return e.check(C.lwse_ds_resident_load(e.h, t)) }

// DsTick applies the DS row patches of one pass of the DS work queue, sweeps every DS and returns
// the DS rows whose decisions changed.  ch.ds_out / role_out / revrole_out are the full output
// tables in engine-owned pinned memory (valid until the next DS call): read a listed DS's rows at its
// role_base / rev_base.
func (e *Engine) DsTick(segs []C.lwse_patch_seg, ch *C.lwse_ds_changes) ([]uint32, error) {
	var p *C.lwse_patch_seg
	if len(segs) > 0 {
		p = &segs[0]
	}
	if err := e.check(C.lwse_ds_resident_tick(e.h, p, C.uint32_t(len(segs)), ch)); err != nil {
		return nil, err
	}
	if ch.n_changed == 0 {
		return nil, nil
	}
	return unsafe.Slice((*uint32)(unsafe.Pointer(ch.ds_rows)), int(ch.n_changed)), nil
}

// DsTickInfo reports how the last DsTick read ready counts: whether it ran linked (a
// LWSE_TABLE_DS_LINKS patch since DsResidentLoad: linked revision-role rows take their child's ready
// count from the most recently submitted LWS tick), the rows that took that value, the linked rows
// that fell back to their own, and the LWS ticks submitted when it read them.
func (e *Engine) DsTickInfo() (C.lwse_ds_tick_info, error) {
	var info C.lwse_ds_tick_info
	err := e.check(C.lwse_ds_resident_tick_info(e.h, &info))
	return info, err
}

// Forecast replays the rest of every DS rollout from the resident DS tables as the last DsTick left
// them, assuming every child becomes ready before each reconcile: per DS the flags, cycles and
// trajectory offset, per role the peak replicas, availability floor and final counts, and (when
// out.steps is set) the {old, new} rows of each step.  It changes no DsTick output and never waits for
// LeaderWorkerSet ticks; a status or kubectl surface reads it, not Reconcile().
func (e *Engine) Forecast(out *C.lwse_ds_forecast_out) error {
	return e.check(C.lwse_ds_resident_forecast(e.h, out))
}

// PlaceWhatIf answers "what would the placement round give with these node and request patches and
// these extra requests?" over the resident tables without changing them: the resident rows whose
// placement would change (with their current and hypothetical rows), the rows of the extra requests,
// and lost / moved / gained counts.  It never waits for or drops a tick.  A validating webhook calls it
// on LWS create / scale-up with an exclusive topology, a kubectl drain planner with cordon segments.
func (e *Engine) PlaceWhatIf(q *C.lwse_place_whatif) error {
	return e.check(C.lwse_resident_place_whatif(e.h, q))
}

// RolloutWhatIf answers "if this LeaderWorkerSet edit were pushed, what would its rollout do?" over the
// resident tables without changing them: per proposal (a resident row and the row the edited object
// would encode to) the controller's first write, and the forecast of the rollout it starts — controller
// writes, peak leader StatefulSet replicas, the ready-group floor, and whether it finishes or stops at
// the spec partition.  It never waits for or drops a tick.  A kubectl plugin or a validating webhook
// calls it on a template, replicas or rollout-settings edit; a fleet image bump asks one proposal per
// object in one call.
func (e *Engine) RolloutWhatIf(q *C.lwse_rollout_whatif) error {
	return e.check(C.lwse_resident_rollout_whatif(e.h, q))
}

// DsRolloutWhatIf answers "if this DisaggregatedSet edit were pushed, what would its rollout do?" over the
// resident DS tables without changing them: per proposal (a DS row, NEW_REVISION for a template edit, ROLES with
// new role rows for a scale or new rollout settings) the DS controller's first decision, read through the child
// links as the DS tick reads them, and the forecast of the rollout it starts — steps, peak replicas and the
// availability floor per role.  It never waits for or drops a tick.  A validating webhook calls it on a DS update;
// a fleet image bump asks one proposal per DS in one call.
func (e *Engine) DsRolloutWhatIf(q *C.lwse_ds_rollout_whatif) error {
	return e.check(C.lwse_resident_ds_rollout_whatif(e.h, q))
}

// DsDrain answers "does draining these nodes or topology domains take an inference service down, or
// stall its rollout?" over the resident LWS and DS tables: the DisaggregatedSets whose linked child
// LeaderWorkerSets lose ready groups, with SERVICE_LOST / OLD_SERVICE_LOST / STALLS verdicts and their
// ds_out rows before and after.  A drain or maintenance controller calls it before cordoning a rack or
// zone, a kubectl drain dry-run plugin to report the services at risk.
func (e *Engine) DsDrain(q *C.lwse_ds_drain_query) error {
	return e.check(C.lwse_resident_ds_drain(e.h, q))
}

// DsDrainCost gives DsDrain's counts for every node (scope LWSE_DRAIN_NODES) or every domain
// (LWSE_DRAIN_DOMAINS) in one call, to rank maintenance candidates.
func (e *Engine) DsDrainCost(scope uint32, out *C.lwse_ds_drain_cost) error {
	return e.check(C.lwse_resident_ds_drain_cost(e.h, C.uint32_t(scope), out))
}

// DrainPlaceCost answers "if I drain this node or this domain, do the groups it restarts find a new
// exclusive domain?" for every node (scope LWSE_DRAIN_NODES) or every domain (LWSE_DRAIN_DOMAINS) in one
// call: restarted groups, unpinned requests, those left without a domain (stranded), others that lose theirs
// (bumped) and the placement what-if's counts.  A maintenance controller ranks the next rack to drain with it.
func (e *Engine) DrainPlaceCost(scope uint32, out *C.lwse_drain_place_cost) error {
	return e.check(C.lwse_resident_drain_place_cost(e.h, C.uint32_t(scope), out))
}

// RolloutPlace answers "do the groups this rollout adds find an exclusive domain?" for a list of resident
// LeaderWorkerSets, or of proposed edits (q.recs), in one call: per entry the forecast's peak, the groups up to it
// that need a request (surge), those left without a domain (stranded) and the other requests that lose theirs.
// An admission webhook or a rollout controller checks an edit with it before pushing it.
func (e *Engine) RolloutPlace(q *C.lwse_rollout_place_query) error {
	return e.check(C.lwse_resident_rollout_place(e.h, q))
}

// RolloutPlaceWaves packs distinct resident LeaderWorkerSets, or proposed edits of them (q.recs), first-fit in the
// order given into at most q.max_waves waves whose rollouts, pushed together, give every group they add an
// exclusive domain (LWSE_RPW_STRANDED) and, with LWSE_RPW_BUMPED, take none from a placed group.  A fleet-wide
// template bump pushes wave 0, waits for its rollouts to finish and calls again with the objects that remain.
func (e *Engine) RolloutPlaceWaves(q *C.lwse_rollout_place_waves_query) error {
	return e.check(C.lwse_resident_rollout_place_waves(e.h, q))
}

// PlaceExplain answers "why is this group not placed?" for rows of a placement round: per row, how many topology
// domains are too small, have no usable node, are held ahead of it in its namespace (and by which row), or are
// open, the domain it falls short in by the fewest slots, and whether cordoned nodes would make one fit.  The
// round is the last tick's, or the what-if round of q's segments and extra rows.  A controller turns a row into
// the Pending event of an exclusive group; an autoscaler or rollout planner explains the rows a query stranded.
func (e *Engine) PlaceExplain(q *C.lwse_place_explain_query) error {
	return e.check(C.lwse_resident_place_explain(e.h, q))
}

// ScaleHeadroom answers "how many replicas can this object go to right now?" for a list of settled exclusive
// LeaderWorkerSets in one call: per entry the largest replicas (up to an optional ceiling, such as the HPA's
// maxReplicas) at which every group the scale-up adds still finds an exclusive domain, and the counters of the
// first replicas that does not.  An autoscaler clamps its desired replicas to max_replicas before it writes the
// scale subresource, so that no group it adds stays Pending.
func (e *Engine) ScaleHeadroom(q *C.lwse_scale_headroom_query) error {
	return e.check(C.lwse_resident_scale_headroom(e.h, q))
}

// DrainWaves packs distinct node rows (scope LWSE_DRAIN_NODES) or domain ids (LWSE_DRAIN_DOMAINS), in the order
// given, first-fit into at most q.max_waves waves whose drain takes no LeaderWorkerSet below its floor.  A
// maintenance controller drains wave 0, waits for recovery and calls again with the keys that remain.
func (e *Engine) DrainWaves(q *C.lwse_drain_waves_query) error {
	return e.check(C.lwse_resident_drain_waves(e.h, q))
}

// DsDrainWaves packs distinct node rows or domain ids, in the order given, first-fit into at most q.max_waves
// waves whose drain triggers none of the verdicts in q.constraints (LWSE_DSW_*): no LeaderWorkerSet below its
// floor, no DisaggregatedSet losing the service of its new or an old revision, no rollout stalled.
func (e *Engine) DsDrainWaves(q *C.lwse_ds_drain_waves_query) error {
	return e.check(C.lwse_resident_ds_drain_waves(e.h, q))
}

// DrainPlaceWaves packs distinct node rows or domain ids, in the order given, first-fit into at most q.max_waves
// waves whose drain triggers none of the verdicts in q.constraints (LWSE_DPW_*): no LeaderWorkerSet below its
// floor, no unpinned request left without a new exclusive domain, and (opt-in) no other request losing its domain.
func (e *Engine) DrainPlaceWaves(q *C.lwse_drain_place_waves_query) error {
	return e.check(C.lwse_resident_drain_place_waves(e.h, q))
}

// GroupKeys computes SHA-1 digests (20 bytes each) of n strings laid out CSR-style.
func (e *Engine) GroupKeys(bytes *C.uint8_t, offsets *C.uint32_t, n uint32, digests *C.uint8_t) error {
	return e.check(C.lwse_group_keys_host(e.h, bytes, offsets, C.uint32_t(n), digests))
}

// --- incremental form: tables resident on the device, fed from watch events -----------------

// ResidentLoad copies the four input tables to the device, where they stay.
func (e *Engine) ResidentLoad(t *LwsTables) error {
	ct := t.c()
	return e.check(C.lwse_resident_load(e.h, &ct))
}

// ResidentPatch overwrites n rows of one resident table (rows[i] <- i-th packed row of values):
// what an informer delta (pod phase change, sts status update, spec edit) turns into.
func (e *Engine) ResidentPatch(which C.lwse_table, rows *C.uint32_t, values unsafe.Pointer, n uint32) error {
	return e.check(C.lwse_resident_patch(e.h, which, rows, values, C.uint32_t(n)))
}

// ResidentSweep sweeps the resident tables and returns only the result rows that changed since
// the previous sweep — the objects whose Reconcile() has something to do.
func (e *Engine) ResidentSweep(flags uint32, ch *C.lwse_changes) error {
	return e.check(C.lwse_resident_sweep(e.h, C.uint32_t(flags), ch))
}

// --- device-pointer form: one reconcile tick (sweep + placement round, concurrently) --------

// ReconcileDevice enqueues one tick on stream (nil = the engine's stream); no synchronize.
func (e *Engine) ReconcileDevice(t *LwsTables, reqs *C.lwse_place_req, n uint32, occupancy *C.uint32_t,
	nNamespaces uint32, placeOut *C.lwse_place_out, stream unsafe.Pointer) error {
	ct := t.c()
	return e.check(C.lwse_reconcile_device(e.h, &ct, reqs, C.uint32_t(n), occupancy, C.uint32_t(nNamespaces), placeOut, stream))
}

// --- one operator replica per GPU of a node: placement parts exchanged over NVLink -----------

// ExchangeCreate allocates this replica's exchange buffer and returns its 64-byte IPC handle;
// the replicas swap handles (any transport) and each calls ExchangeConnect with all of them.
func (e *Engine) ExchangeCreate(reqsPerPart, world, rank uint32) ([64]byte, error) {
	var h [64]byte
	err := e.check(C.lwse_exchange_create(e.h, C.uint32_t(reqsPerPart), C.uint32_t(world), C.uint32_t(rank), unsafe.Pointer(&h[0])))
	return h, err
}

func (e *Engine) ExchangeConnect(handles []byte) error {
	return e.check(C.lwse_exchange_connect(e.h, unsafe.Pointer(&handles[0])))
}

// ReconcileExchangedDevice: a tick of one shard; localPart = [occupancy | request rows] in device memory.
func (e *Engine) ReconcileExchangedDevice(t *LwsTables, localPart unsafe.Pointer, nNamespaces uint32,
	placeOut *C.lwse_place_out, stream unsafe.Pointer) error {
	ct := t.c()
	return e.check(C.lwse_reconcile_exchanged_device(e.h, &ct, localPart, C.uint32_t(nNamespaces), placeOut, stream))
}
