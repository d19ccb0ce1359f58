/*
 * lwse.h — C ABI of the H100 reconcile-and-placement engine ("lwse") for the
 * LeaderWorkerSet / DisaggregatedSet controllers.
 *
 * This is the drop-in boundary for the hot path named in BASELINE.json:
 * a cgo (or any FFI) caller hands fixed-width record tables to the engine and
 * reads fixed-width result tables back.  Plain pointers and sizes only; no
 * CUDA, torch or C++ types cross this boundary.
 *
 * The reference (kubernetes-sigs/lws @ 1d9204a2) has no FFI for this path —
 * every hot function is package-private Go.  Each entry point below therefore
 * cites the reference function(s) whose arithmetic it replaces
 * (paths relative to the reference root):
 *
 *   lwse_sweep_lws_*   pkg/controllers/leaderworkerset_controller.go:280-373
 *                      (rollingUpdateParameters), :414-509 (updateConditions),
 *                      :576-641 (getReplicaStates), :643-708 (partition math),
 *                      :811-830 (stsMaxUnavailable);
 *                      pkg/controllers/pod_controller.go:100-172 (worker-sts
 *                      gating), :204-266 (handleRestartPolicy), :268-295
 *                      (workerPodBelongsToLeader), :315-336
 *                      (topologyValueFromPod), :338-362 (pendingPodsInGroup),
 *                      :434-443 (worker ordinals);
 *                      pkg/schedulerprovider/volcano_provider.go:72-83 (MinMember)
 *   lwse_place_*       build-defined placement spec over the constraints of
 *                      pkg/webhooks/pod_webhook.go:185-227 (exclusive affinity /
 *                      anti-affinity per topology domain) — the reference has no
 *                      node scoring; see DESIGN.md "Placement (parity unpinned)"
 *   lwse_sweep_ds_*    pkg/controllers/disaggregatedset/planner.go:61-352,
 *                      executor.go:199-302 (planner state / config / stability),
 *                      :330-398 (scaleDownOld), disaggregatedset_controller.go:
 *                      203-236 (cleanup predicate), service_manager.go:57-89
 *   lwse_ds_resident_* the same arithmetic over resident DS tables, fed by DS and child-LWS
 *                      watch events (disaggregatedset_controller.go:55-126, :273)
 *   lwse_resident_rollout_whatif  the sweep and the forecast above over a proposed LWS row: the
 *                      encoder's leaderWorkerSetUpdated (leaderworkerset_controller.go:150-159,
 *                      :325-332) into rollingUpdateParameters (:280-373), Case 4 (:351-361)
 *   lwse_resident_ds_rollout_whatif  the DS sweep and forecast above over the rows a proposed DS edit
 *                      encodes to: a new ComputeRevision(spec.roles) (utils.go:173-199) retires the
 *                      target revision into the old ones (GroupByRevision, utils.go:192-211)
 *   lwse_resident_drain_*  pod_controller.go:204-266 (handleRestartPolicy), :268-295, :338-362 over
 *                      the resident tables with the pods of drained nodes deleting;
 *                      lwse_resident_drain_budget* adds a build-defined availability floor from
 *                      leaderworkerset_controller.go:302 (the reference has no drain budget)
 *   lwse_resident_ds_drain*  the drain budget's lost groups through the DS links into the DS sweep:
 *                      service_manager.go:57-89, :174-189 (serving), executor.go:270-281 (stable)
 *   lwse_group_keys_*  pkg/webhooks/pod_webhook.go:180-182 + pkg/utils/utils.go:39-43
 *                      (SHA-1 group / subgroup keys)
 *   lwse_subgroup_keys_*  pkg/webhooks/pod_webhook.go:249-255 (getSubGroupIndex) + :130,:151
 *                      (the subgroup key of that index)
 *
 * Conventions
 *   - All records are little-endian plain-old-data with explicit padding; every
 *     table base must be 16-byte aligned.
 *   - Every function returns LWSE_OK (0) or a negative lwse_status.  Nothing
 *     aborts.  lwse_last_cuda_error() returns the cudaError_t behind
 *     LWSE_ERR_CUDA.
 *   - The caller owns every host buffer (cgo: C.malloc / pinned pool — the
 *     engine never retains a host pointer past the call).  The engine owns its
 *     device staging memory.
 *   - An engine handle is bound to one CUDA device and runs one sweep at a time
 *     (internal mutex).  Create one per GPU.
 *   - There is no CPU fallback: if no CUDA device is usable lwse_create fails
 *     with LWSE_ERR_NO_DEVICE.
 */
#ifndef LWSE_H_
#define LWSE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LWSE_ABI_VERSION 2u

#if defined(__GNUC__)
#define LWSE_API __attribute__((visibility("default")))
#else
#define LWSE_API
#endif

/* ------------------------------------------------------------------------- */
/* Status codes                                                              */
/* ------------------------------------------------------------------------- */
typedef enum lwse_status {
  LWSE_OK = 0,
  LWSE_ERR_INVALID_ARG = -1, /* NULL / misaligned pointer, bad count            */
  LWSE_ERR_NO_DEVICE = -2,   /* no usable CUDA device (no CPU fallback exists)  */
  LWSE_ERR_CUDA = -3,        /* a CUDA call failed; see lwse_last_cuda_error    */
  LWSE_ERR_OOM = -4,         /* device or pinned allocation failed              */
  LWSE_ERR_BAD_TABLE = -5,   /* a base/count in a record points outside a table */
  LWSE_ERR_NOT_READY = -6,   /* e.g. lwse_place_* before lwse_upload_nodes      */
  LWSE_ERR_UNSUPPORTED = -7  /* e.g. more than LWSE_DS_MAX_ROLES roles          */
} lwse_status;

/* ------------------------------------------------------------------------- */
/* Input records                                                             */
/* ------------------------------------------------------------------------- */

#define LWSE_NONE 0xFFFFFFFFu           /* "no index" (unscheduled, no domain, …) */
#define LWSE_NODE_NOT_FOUND 0xFFFFFFFEu /* leader.spec.nodeName set, Node object missing */

/* One LeaderWorkerSet object (64 B).  The first 16 bytes are everything the
 * per-group kernel needs from its owner. */
typedef struct lwse_lws_rec {
  uint64_t rev_hash;  /* hash of the revisionKey handed to the reconciler
                         (leaderworkerset_controller.go:159,:196)                */
  int32_t size;       /* *spec.leaderWorkerTemplate.size                         */
  uint32_t flags;     /* LWSE_LWS_* */
  int32_t replicas;   /* *spec.replicas                                          */
  int32_t partition;  /* *spec.rolloutStrategy.rollingUpdateConfiguration.partition */
  int32_t max_surge;  /* IntVal, or the percent number when ..._IS_PERCENT       */
  int32_t max_unavailable;
  int32_t sts_replicas;            /* leader sts *spec.replicas                  */
  int32_t sts_partition;           /* leader sts rollingUpdate.partition         */
  int32_t sts_replicas_annotation; /* Atoi(leaderworkerset.sigs.k8s.io/replicas) */
  int32_t subgroup_size;           /* 0 = no subGroupPolicy                      */
  uint64_t uid_hash;  /* hash of metadata.uid: shard key, placement priority     */
  uint32_t group_base;             /* first row of this object in the group table */
  uint32_t group_count;            /* rows = group indices 0..group_count-1      */
} lwse_lws_rec;

#define LWSE_LWS_SURGE_IS_PERCENT (1u << 0)
#define LWSE_LWS_UNAVAIL_IS_PERCENT (1u << 1)
#define LWSE_LWS_STS_EXISTS (1u << 2)       /* leader StatefulSet found (:293)            */
#define LWSE_LWS_UPDATED (1u << 3)          /* leaderWorkerSetUpdated argument (:325)     */
#define LWSE_LWS_ANNOT_VALID (1u << 4)      /* strconv.Atoi of the annotation ok (:351)   */
#define LWSE_LWS_RESTART_SHIFT 5            /* 2 bits: lwse_restart_policy                */
#define LWSE_LWS_RESTART_MASK (3u << 5)
#define LWSE_LWS_RECREATE_AFTER_START_ANNOT (1u << 7) /* pod_controller.go:220            */
#define LWSE_LWS_STARTUP_LEADER_READY (1u << 8)       /* spec.startupPolicy == LeaderReady */
#define LWSE_LWS_EXCLUSIVE_TOPOLOGY (1u << 9) /* exclusive-topology annotation present    */
#define LWSE_LWS_SUBGROUP_LEADER_EXCLUDED (1u << 10)
#define LWSE_LWS_GROUP_LABEL_INVALID (1u << 11) /* a leader pod's group-index label fails
                                                   Atoi → updateConditions error (:434)   */
#define LWSE_LWS_INTSTR_INVALID (1u << 12)  /* maxSurge/maxUnavailable string not "N%"    */
#define LWSE_LWS_IRREGULAR (1u << 13)       /* encoder could not express the object
                                               (see DESIGN.md "Encoder invariants")       */

typedef enum lwse_restart_policy {
  LWSE_RESTART_NONE = 0,          /* "None", "Default", anything else            */
  LWSE_RESTART_ON_POD_RESTART = 1,/* RecreateGroupOnPodRestart                   */
  LWSE_RESTART_AFTER_START = 2    /* RecreateGroupAfterStart                     */
} lwse_restart_policy;

/* One pod group = leader pod slot + its worker StatefulSet (64 B).
 * Row r of an object describes group index r. */
typedef struct lwse_group_rec {
  uint64_t leader_rev_hash;   /* leader pod template-revision-hash label          */
  uint64_t wsts_rev_hash;     /* worker sts template-revision-hash label          */
  int32_t wsts_spec_replicas; /* worker sts *spec.replicas                        */
  int32_t wsts_avail_replicas;/* worker sts status.availableReplicas              */
  uint32_t leader_uid_hash;   /* leader pod metadata.uid                          */
  uint32_t wsts_uid_hash;     /* worker sts metadata.uid                          */
  uint32_t wsts_owner_uid_hash; /* controller ownerRef.uid of the worker sts      */
  uint32_t leader_node;       /* node-table row, LWSE_NONE, or LWSE_NODE_NOT_FOUND */
  uint32_t pod_base;          /* first row of this group in the pod columns       */
  uint32_t pod_count;         /* pods carrying (set name, group index) labels     */
  uint32_t lws_index;         /* row of the owning object in the LWS table        */
  uint32_t flags;             /* LWSE_GRP_* */
  uint32_t reserved[2];
} lwse_group_rec;

#define LWSE_GRP_POD_PRESENT (1u << 0)    /* a leader pod with this group-index label exists */
#define LWSE_GRP_POD_NAME_MATCH (1u << 1) /* its name == "<lws>-<idx>" (:609)                 */
#define LWSE_GRP_POD_RUNNING (1u << 2)    /* status.phase == Running                          */
#define LWSE_GRP_POD_READY (1u << 3)      /* Ready condition == True                          */
#define LWSE_GRP_POD_DELETING (1u << 4)   /* deletionTimestamp != nil                         */
#define LWSE_GRP_WSTS_LABEL_NAME_MATCH (1u << 5) /* sts with this group-index label is named
                                                    "<lws>-<idx>" (:611)                      */
#define LWSE_GRP_WSTS_FOUND (1u << 6)     /* Get(sts named like the leader pod) succeeded     */
#define LWSE_GRP_WSTS_REV_SETTLED (1u << 7) /* status.currentRevision == status.updateRevision */
#define LWSE_GRP_WSTS_OWNER_IS_POD (1u << 8)
#define LWSE_GRP_WSTS_OWNER_NAME_MATCH (1u << 9) /* sts ownerRef.name == leader pod name      */
#define LWSE_GRP_MISTAKEN_ANNOTATION (1u << 10)  /* leader carries leader-name annotation     */
#define LWSE_GRP_REVISION_EXISTS (1u << 11)      /* ControllerRevision for leader's key found */

/* Pods are stored column-split: the per-sweep-hot state BYTE (changes with every status
 * update; the only pod column a sweep streams) and the cold identity row (16 B, 16-byte
 * aligned; fixed at pod creation apart from the node binding; read only for pods that have a
 * restart / deletion event, and by the optional occupancy count). */
typedef uint8_t lwse_pod_state; /* LWSE_POD_* */

typedef struct lwse_pod_ident { /* 16 B */
  uint64_t rev_hash;       /* template-revision-hash label (hash64)                  */
  uint32_t owner_uid_hash; /* controller ownerRef.uid — a 32-bit hash: two different UIDs
                              compare equal with probability 2^-32 per comparison (only
                              pods that already have a restart event are ever compared;
                              DESIGN.md "hash widths")                                */
  uint32_t place;          /* LWSE_PODID_* | node << LWSE_PODID_NODE_SHIFT            */
} lwse_pod_ident;

#define LWSE_POD_PHASE_MASK 3u       /* 0 other, 1 Pending, 2 Running              */
#define LWSE_POD_PHASE_PENDING 1u
#define LWSE_POD_PHASE_RUNNING 2u
#define LWSE_POD_ANY_RESTART (1u << 2) /* some (init)containerStatus.restartCount > 0 */
#define LWSE_POD_DELETING (1u << 3)
#define LWSE_POD_OWNER_SHIFT 4       /* 2 bits: 0 none, 1 Pod, 2 StatefulSet, 3 other */
#define LWSE_POD_OWNER_MASK (3u << 4)
#define LWSE_POD_OWNER_NAME_MATCH (1u << 6) /* ownerRef.name == "<lws>-<group>"    */
#define LWSE_POD_IS_LEADER (1u << 7) /* worker-index label == "0"                  */

#define LWSE_PODID_NAME_OK (1u << 0)   /* GetParentNameAndOrdinal ordinal != -1    */
#define LWSE_PODID_SCHEDULED (1u << 1) /* node field below is valid                */
#define LWSE_PODID_NODE_SHIFT 10       /* 22-bit node-table row                    */
#define LWSE_POD_NODE_MAX ((1u << 22) - 1u)

/* One node (16 B). */
typedef struct lwse_node_rec {
  uint64_t topo_value_hash; /* hash of node.labels[topologyKey]                   */
  uint32_t domain_id;       /* dense id of that label value, or LWSE_NONE         */
  uint16_t capacity;        /* pod slots available to LWS pods                    */
  uint16_t flags;           /* LWSE_NODE_* */
} lwse_node_rec;

#define LWSE_NODE_HAS_TOPOLOGY (1u << 0) /* label present (pod_controller.go:330) */
#define LWSE_NODE_SCHEDULABLE (1u << 1)

/* ------------------------------------------------------------------------- */
/* Output records                                                            */
/* ------------------------------------------------------------------------- */

/* Per LeaderWorkerSet (32 B). */
typedef struct lwse_lws_out {
  int32_t sts_partition;      /* rollingUpdateParameters → stsPartition           */
  int32_t sts_replicas;       /* rollingUpdateParameters → replicas               */
  int32_t sts_max_unavailable;/* constructLeaderStatefulSetApplyConfiguration     */
  int32_t ready_replicas;     /* status.readyReplicas                             */
  int32_t updated_replicas;   /* status.updatedReplicas                           */
  int32_t min_member;         /* PodGroup spec.minMember                          */
  uint32_t flags;             /* LWSE_LOUT_* */
  int32_t unready_replicas;   /* calculateLWSUnreadyReplicas (diagnostic; 0 when
                                 the reference does not compute it)               */
} lwse_lws_out;

#define LWSE_LOUT_RUP_ERROR (1u << 0)     /* rollingUpdateParameters returned err  */
#define LWSE_LOUT_STATUS_ERROR (1u << 1)  /* updateConditions returned err         */
#define LWSE_LOUT_COND_SHIFT 2            /* 2 bits: lwse_condition                */
#define LWSE_LOUT_COND_MASK (3u << 2)
#define LWSE_LOUT_UPDATE_DONE (1u << 4)
#define LWSE_LOUT_EVENT_SHIFT 5           /* 2 bits: lwse_surge_event              */
#define LWSE_LOUT_EVENT_MASK (3u << 5)
#define LWSE_LOUT_IRREGULAR (1u << 7)
#define LWSE_LOUT_BAD_TABLE (1u << 8)     /* group_base/group_count outside the group table */

typedef enum lwse_condition {
  LWSE_COND_PROGRESSING = 0,
  LWSE_COND_AVAILABLE = 1,
  LWSE_COND_UPDATE_IN_PROGRESS = 2 /* UpdateInProgress + Progressing              */
} lwse_condition;

typedef enum lwse_surge_event {
  LWSE_EVENT_NONE = 0,
  LWSE_EVENT_DELETE_ONE = 1,  /* "deleting surge replica %s-%d" (:314)            */
  LWSE_EVENT_DELETE_RANGE = 2 /* "deleting surge replicas from … to …" (:316)     */
} lwse_surge_event;

/* Per pod group (16 B). */
typedef struct lwse_group_out {
  uint32_t flags;           /* LWSE_GOUT_* */
  uint32_t first_trigger;   /* pod row (relative to pod_base) of the first pod
                               whose reconcile would recreate the group, or NONE  */
  int32_t worker_replicas;  /* worker sts replicas (= size-1, ordinals start at 1)
                               when LWSE_GOUT_CREATE_WSTS, else 0                 */
  uint32_t domain_id;       /* nodeSelector topology domain of the workers
                               (topologyValueFromPod), or LWSE_NONE               */
} lwse_group_out;

#define LWSE_GOUT_STATE_READY (1u << 0)    /* getReplicaStates ready  (name-checked)   */
#define LWSE_GOUT_STATE_UPDATED (1u << 1)  /* getReplicaStates updated                 */
#define LWSE_GOUT_COUNTED (1u << 2)        /* leader pod visited by updateConditions   */
#define LWSE_GOUT_COND_READY (1u << 3)     /* updateConditions ready                   */
#define LWSE_GOUT_COND_UPDATED (1u << 4)   /* updateConditions updated                 */
#define LWSE_GOUT_PENDING (1u << 5)        /* pendingPodsInGroup                       */
#define LWSE_GOUT_DELETE_LEADER (1u << 6)  /* some pod's reconcile issues Delete(leader) */
#define LWSE_GOUT_LEADER_DELETING (1u << 7)/* …returns true because it is already going  */
#define LWSE_GOUT_RESTART_ERROR (1u << 8)  /* worker name failed to parse (:231)       */
#define LWSE_GOUT_CREATE_WSTS (1u << 9)    /* leader reconcile reaches Create(worker sts) */
#define LWSE_GOUT_WAIT_SCHEDULE (1u << 10) /* exclusive topology, leader unscheduled   */
#define LWSE_GOUT_TOPOLOGY_ERROR (1u << 11)/* node lacks the topology label (:331)     */
#define LWSE_GOUT_REQUEUE_REVISION (1u << 12) /* revision missing → requeue 1s (:152)  */
#define LWSE_GOUT_CREATE_PODGROUP (1u << 13)  /* SchedulerProvider.CreatePodGroupIfNotExists reached */
#define LWSE_GOUT_BAD_TABLE (1u << 14)     /* lws_index / pod_base+pod_count outside a table  */

/* ------------------------------------------------------------------------- */
/* Table bundles                                                             */
/* ------------------------------------------------------------------------- */

/* The same bundle is used with host pointers (lwse_sweep_lws_host) and with
 * device pointers (lwse_sweep_lws_device). */
typedef struct lwse_lws_tables {
  const lwse_lws_rec* lws;
  uint32_t n_lws;
  const lwse_group_rec* groups;
  uint32_t n_groups;
  const lwse_pod_state* pod_state; /* n_pods words  */
  const lwse_pod_ident* pod_ident; /* n_pods rows   */
  uint64_t n_pods;
  lwse_lws_out* lws_out;     /* n_lws rows   */
  lwse_group_out* group_out; /* n_groups rows */
  uint32_t* node_occupancy;  /* optional: n_nodes counters, scheduled pods per node
                                over the whole pod table (the call overwrites
                                them; it reads the identity column for it); NULL
                                to skip                                           */
  uint32_t flags;            /* LWSE_SWEEP_* */
} lwse_lws_tables;

#define LWSE_SWEEP_GANG (1u << 0) /* a SchedulerProvider is configured (min_member,
                                     CREATE_PODGROUP are meaningful)              */
#define LWSE_SWEEP_SKIP_GROUP_PASS (1u << 1) /* profiling: run only the LWS-level pass
                                                (group_out must hold a previous result) */
#define LWSE_SWEEP_SKIP_LWS_PASS (1u << 2)   /* profiling: skip the LWS-level pass       */
#define LWSE_SWEEP_REUSE_POD_IDENT (1u << 4) /* host entry point only: the pod identity column
                                                (revision hash, owner uid — fixed at pod creation)
                                                is unchanged since this engine's previous host
                                                sweep with the same n_pods; skip its upload     */
#define LWSE_SWEEP_PLACE_GROUPED (1u << 5)   /* lwse_reconcile_*_device: the placement requests are grouped by
                                                namespace (ns non-decreasing) — enables the namespace-parallel
                                                placement kernels (one CTA per namespace, state in shared memory).
                                                A promise: a violated order is counted, rows are then unspecified  */
#define LWSE_SWEEP_PLACE_SCAN (1u << 6)      /* with GROUPED: brute-force (request x node) scoring from the
                                                TMA-staged node table instead of the two-level search (same rows) */
#define LWSE_SWEEP_SKIP_POD_SCAN (1u << 3)   /* profiling: skip the pod-state scan (its
                                                bitmaps must hold a previous result)     */

typedef struct lwse_config {
  uint32_t abi_version; /* LWSE_ABI_VERSION */
  int32_t device;       /* CUDA device ordinal */
  uint32_t flags;       /* reserved, 0 */
  uint32_t reserved;
} lwse_config;

typedef struct lwse_engine lwse_engine;

/* ------------------------------------------------------------------------- */
/* Lifecycle                                                                 */
/* ------------------------------------------------------------------------- */
LWSE_API int lwse_create(const lwse_config* cfg, lwse_engine** out);
LWSE_API void lwse_destroy(lwse_engine* e);
LWSE_API const char* lwse_strerror(int status);
LWSE_API int lwse_last_cuda_error(const lwse_engine* e);
LWSE_API uint32_t lwse_abi_version(void);
/* The CUDA stream (cudaStream_t) all of this engine's work is issued on. */
LWSE_API void* lwse_stream(const lwse_engine* e);
/* Number of kernels this engine has launched since creation. */
LWSE_API uint64_t lwse_launch_count(const lwse_engine* e);

/* Shard an object onto one of n engines (Go: hash(LWS.UID) mod nGPU; DS-owned
 * LWS pass the DS uid hash so a DS and its children co-reside). */
LWSE_API uint32_t lwse_shard_of(uint64_t uid_hash, uint32_t n_shards);
/* The 64-bit string hash the encoders use for revision keys / label values /
 * UIDs (FNV-1a 64; 32-bit fields take the low word xor the high word). */
LWSE_API uint64_t lwse_hash64(const void* bytes, size_t len);

/* ------------------------------------------------------------------------- */
/* Node table                                                                */
/* ------------------------------------------------------------------------- */
/* Copies n node rows to the device; they stay resident across sweeps (and are patched row by row
 * with LWSE_TABLE_NODES).  After lwse_resident_load, the occupancy counters of the resident pods are
 * recounted for the new table. */
LWSE_API int lwse_upload_nodes(lwse_engine* e, const lwse_node_rec* nodes, uint32_t n_nodes,
                               uint32_t n_domains);

/* ------------------------------------------------------------------------- */
/* LWS sweep                                                                 */
/* ------------------------------------------------------------------------- */
/* Host buffers in, host buffers out: H2D of the three tables, the sweep
 * kernels, D2H of the two result tables, then a stream synchronize. */
LWSE_API int lwse_sweep_lws_host(lwse_engine* e, const lwse_lws_tables* host_tables);
/* All pointers are device pointers on the engine's device; kernels are
 * enqueued on `stream` (cudaStream_t; NULL = the engine's stream) and the call
 * returns without synchronizing. */
LWSE_API int lwse_sweep_lws_device(lwse_engine* e, const lwse_lws_tables* dev_tables, void* stream);

/* ------------------------------------------------------------------------- */
/* Resident tables: incremental operation                                    */
/* ------------------------------------------------------------------------- */
/* A controller sees watch events, not tables: between two sweeps only a few rows change.
 * The engine can keep the input tables resident in HBM; the host then sends row patches
 * (lwse_resident_patch) and reads back only the result rows that changed
 * (lwse_resident_sweep) — the actions the reconcilers have to take. */
typedef enum lwse_table {
  LWSE_TABLE_LWS = 0,       /* lwse_lws_rec    */
  LWSE_TABLE_GROUPS = 1,    /* lwse_group_rec  */
  LWSE_TABLE_POD_STATE = 2, /* lwse_pod_state  */
  LWSE_TABLE_POD_IDENT = 3, /* lwse_pod_ident  */
  LWSE_TABLE_PLACE_REQS = 4, /* lwse_place_req (lwse_resident_place_load)  */
  LWSE_TABLE_NODES = 5,       /* lwse_node_rec: the table of the last lwse_upload_nodes.  Rows must be
                                 < its n_nodes: patches never change the table's size, so the caller
                                 reserves spare rows (flags = 0: no request can use them) at upload.
                                 A patched row means what an uploaded row means: a node is usable iff
                                 SCHEDULABLE, HAS_TOPOLOGY and domain_id < n_domains.  Multi-rank
                                 ticks (LWSE_TICK_SHARED_OCCUPANCY): every rank applies the same node
                                 patches in the same tick.                                      */
  LWSE_TABLE_DS = 6,          /* lwse_ds_rec, lwse_ds_role_rec, lwse_ds_revrole_rec: the resident DS   */
  LWSE_TABLE_DS_ROLES = 7,    /* tables (lwse_ds_resident_load).  Only lwse_ds_resident_tick takes     */
  LWSE_TABLE_DS_REVROLES = 8, /* them; lwse_resident_patch / _tick reject them as any unknown table  */
  LWSE_TABLE_DS_LINKS = 9     /* lwse_ds_link, one row per revision-role row (see lwse_ds_link); the
                                 same rules as the three DS tables                                  */
} lwse_table;

/* Result rows that differ from the previous resident sweep (all rows after a load).
 * n_* is the number of changed rows; if it exceeds the capacity the surplus rows are not
 * returned and the caller falls back to lwse_resident_outputs.  Order is unspecified. */
typedef struct lwse_changes {
  uint32_t* lws_rows;        /* [lws_capacity]   row numbers          */
  lwse_lws_out* lws_out;     /* [lws_capacity]   their new results    */
  uint32_t lws_capacity;
  uint32_t n_lws;            /* out */
  uint32_t* group_rows;      /* [group_capacity] */
  lwse_group_out* group_out; /* [group_capacity] */
  uint32_t group_capacity;
  uint32_t n_groups;         /* out */
} lwse_changes;

/* Copy the four input tables of `host` to the device; they stay resident (and the
 * previous results are forgotten).  Output pointers in `host` are ignored. */
LWSE_API int lwse_resident_load(lwse_engine* e, const lwse_lws_tables* host);
/* Overwrite n rows of a resident table: row rows[i] ← the i-th packed row of `values` (rows
 * distinct).  Synchronous convenience form of one patch segment of lwse_resident_tick. */
LWSE_API int lwse_resident_patch(lwse_engine* e, lwse_table which, const uint32_t* rows, const void* values,
                                 uint32_t n);
/* Sweep the resident tables (flags: LWSE_SWEEP_GANG).  `changes` may be NULL. */
LWSE_API int lwse_resident_sweep(lwse_engine* e, uint32_t flags, lwse_changes* changes);
/* Every result row of the last resident sweep. */
LWSE_API int lwse_resident_outputs(lwse_engine* e, lwse_lws_out* lws_out, lwse_group_out* group_out);

/* ---- the resident tick: what one pass of the controllers' work queues maps to ---------------
 * Watch events in (as row patches), actions out (the result rows that changed), ONE call:
 *   patches -> scatter kernel -> fused pod scan + group pass -> LWS pass     (engine stream)
 *           \-> placement round over the resident request table            (side stream)
 * The patch rows / values are consumed where the host wrote them when they lie in the engine's
 * arena (pinned, mapped memory: lwse_resident_arena) — no staging copy (large sets go to a device
 * mirror with one copy-engine transfer, small ones are read in place over PCIe); the kernels
 * append the changed result rows to device lists, a publish kernel copies them into pinned,
 * mapped result buffers and raises a sequence word the call spins on: no stream synchronize, no
 * device->host copy-engine launch on the path.  A tick that follows one still in flight is
 * replayed as one CUDA graph (LWSE_TICK_GRAPH=0 turns that off).  Replaces, per reconcile pass, the
 * informer-cache reads of
 * leaderworkerset_controller.go:421,584,598 and pod_controller.go:348 (List) for every object. */

typedef struct lwse_place_req lwse_place_req; /* defined below (Placement) */
typedef struct lwse_place_out lwse_place_out;

/* One patch segment. */
typedef struct lwse_patch_seg {
  uint32_t table;       /* lwse_table                                                      */
  uint32_t flags;       /* LWSE_PATCH_*                                                    */
  uint32_t n;           /* rows patched                                                    */
  uint32_t first_row;   /* LWSE_PATCH_RANGE: rows first_row .. first_row + n - 1           */
  const uint32_t* rows; /* n distinct row numbers (ignored for a range)                    */
  const void* values;   /* n packed rows of the table's record type                        */
} lwse_patch_seg;

#define LWSE_PATCH_RANGE (1u << 0) /* contiguous rows: one DMA copy instead of a scatter (use it
                                      when a large share of a column changed)              */
#define LWSE_TICK_MAX_SEGS 8u

typedef struct lwse_tick {
  /* in */
  const lwse_patch_seg* segs;
  uint32_t n_segs;
  uint32_t flags; /* LWSE_SWEEP_GANG | LWSE_TICK_* */
  /* out: views of engine-owned pinned memory, valid until the next lwse_resident_* call on this
   * engine.  n_* counts every changed row; rows beyond the capacity (= table size, so this
   * cannot happen for the sweep) are not listed.  Order is unspecified. */
  const uint32_t* lws_rows;
  const lwse_lws_out* lws_out;
  uint32_t n_lws;
  uint32_t n_groups;
  const uint32_t* group_rows;
  const lwse_group_out* group_out;
  const uint32_t* place_rows; /* request rows whose placement changed (LWSE_TICK_PLACE) */
  const lwse_place_out* place_out;
  uint32_t n_place;
  uint32_t place_rounds;
} lwse_tick;

#define LWSE_TICK_PLACE (1u << 8)     /* run the placement round over the resident request table */
#define LWSE_TICK_NO_SWEEP (1u << 9)  /* patches (+ placement) only */
#define LWSE_TICK_SHARED_OCCUPANCY (1u << 10) /* multi-rank: the round runs as lwse_reconcile_shared_device does
                                                 — the engine's occupancy counters are pushed to the peers
                                                 (lwse_exchange_*), the resident requests are solved against
                                                 the sum; combine with LWSE_EXCHANGE_LAGGED                    */
/* (LWSE_SWEEP_PLACE_SCAN selects the brute-force form of the round; the resident request table
 * is checked for namespace grouping when it is loaded) */

/* The engine's patch arena: at least min_bytes of pinned, mapped host memory (grown on demand;
 * growing invalidates the previous base).  Patch segments whose rows / values pointers lie inside
 * it are consumed in place; others are first copied into it by the call. */
LWSE_API int lwse_resident_arena(lwse_engine* e, uint64_t min_bytes, void** base_out, uint64_t* bytes_out);
/* Make the placement request table resident (rows are then patched with LWSE_TABLE_PLACE_REQS);
 * the per-node occupancy the rounds use is counted by the engine from the resident identity
 * column and follows its patches.  Needs lwse_upload_nodes and lwse_resident_load first. */
LWSE_API int lwse_resident_place_load(lwse_engine* e, const lwse_place_req* reqs, uint32_t n_reqs,
                                      uint32_t n_namespaces);
LWSE_API int lwse_resident_tick(lwse_engine* e, lwse_tick* t);
/* The same tick in two halves, for callers that keep the work queue flowing: _submit enqueues a
 * tick and returns at once, _wait blocks (spins on the tick's sequence word) for the OLDEST
 * submitted tick and fills t's outputs.  At most two ticks are in flight (a third _submit returns
 * LWSE_ERR_NOT_READY): while the GPU sweeps tick k the copy engine already moves the patches of
 * tick k+1.  Rules: the patch segments of a tick in flight stay untouched in the arena until its
 * _wait returned (use two arena regions alternately); a tick's output views stay valid until the
 * second _submit after its _wait; every other lwse_resident_* call first waits for (and drops the
 * results of) the ticks in flight.  lwse_resident_tick == _submit + _wait. */
LWSE_API int lwse_resident_tick_submit(lwse_engine* e, const lwse_tick* t);
LWSE_API int lwse_resident_tick_wait(lwse_engine* e, lwse_tick* t);
/* Every placement row of the last tick with LWSE_TICK_PLACE / the occupancy counters the engine
 * maintains (n_nodes words). */
LWSE_API int lwse_resident_place_outputs(lwse_engine* e, lwse_place_out* out);
LWSE_API int lwse_resident_occupancy(lwse_engine* e, uint32_t* occupancy_out);

/* How the most recently submitted tick ran (read-only; nothing waits).  A request table grouped by
 * namespace runs the namespace-parallel form; one that is not (a patch moved a request to another
 * namespace) runs the same form through a namespace index the device builds, rebuilt by the ticks
 * whose patches change a request's namespace.  The general form only runs where the namespace form
 * cannot: too many domains for one CTA's shared memory. */
typedef struct lwse_tick_info {
  uint32_t place_form;  /* LWSE_TICK_FORM_*                                                   */
  uint32_t indexed;     /* 1: the namespace form read the requests through the namespace index */
  uint32_t index_built; /* 1: this tick (re)built that index                                  */
  uint32_t graph;       /* 1: the tick was replayed as a CUDA graph                           */
} lwse_tick_info;
#define LWSE_TICK_FORM_NONE 0u      /* no placement round (no LWSE_TICK_PLACE)               */
#define LWSE_TICK_FORM_GENERAL 1u   /* the general form (+ a diff kernel)                    */
#define LWSE_TICK_FORM_NAMESPACE 2u /* namespace-parallel, two-level                         */
#define LWSE_TICK_FORM_SCAN 3u      /* namespace-parallel, scan (LWSE_SWEEP_PLACE_SCAN)       */
LWSE_API int lwse_resident_tick_info(lwse_engine* e, lwse_tick_info* info);

/* What the node-row patches (LWSE_TABLE_NODES) of the most recently submitted tick did (read-only).
 * The placement round reads the usable nodes through a domain-sorted index on the device.  A patch
 * that only changes a node's capacity keeps the index; one that changes whether a node is usable,
 * or the domain of a usable node, has the next placement round rebuild it first (three kernels in
 * front of the round). */
typedef struct lwse_node_info {
  uint32_t rows_patched; /* node rows in the tick's segments                                      */
  uint32_t index_built;  /* 1: this tick rebuilt the node index                                    */
  uint32_t n_usable;     /* usable nodes after the tick's patches                                  */
  uint32_t reserved;
} lwse_node_info;
LWSE_API int lwse_resident_node_info(lwse_engine* e, lwse_node_info* info);

/* ---- rolling-update forecast ----------------------------------------------------------------
 * The rest of every LeaderWorkerSet rolling update, replayed on the device from the current LWS rows
 * and group results: the controller writes (partition, replicas) to the leader StatefulSet
 * (rollingUpdateParameters, leaderworkerset_controller.go:280-373, with the partition walk :643-673),
 * and the model is an ideal StatefulSet controller and kubelet: after each write every group the
 * StatefulSet would roll is ready.  The replay runs on a private copy of the object's flag bytes (the
 * low five bits of lwse_group_out.flags: STATE_READY, STATE_UPDATED, COUNTED, COND_READY, COND_UPDATED).
 *
 * An object has C = max(group_count, sts_replicas, replicas + surge) slots, surge being maxSurge scaled
 * and clamped to [0, replicas] (:307); slot idx < group_count starts as group idx's flag byte, the
 * others (room for surge groups) at 0.  One cycle:
 *   1. pass: the LWS pass of lwse_sweep_lws_* (the same device code) over the private row and slots
 *      gives (p', n') = (sts_partition, sts_replicas) and the status;
 *   2. apply: the row takes STS_EXISTS, ANNOT_VALID, sts_replicas = n', sts_partition = p',
 *      sts_replicas_annotation = replicas and loses UPDATED (what the server-side apply writes,
 *      :375-411, :831-853); slot idx >= n' becomes 0 (the group is gone); slot idx < n' becomes
 *      STATE_READY|COUNTED|COND_READY, plus STATE_UPDATED|COND_UPDATED when idx >= p' or the old byte
 *      had COND_UPDATED (only ordinals >= partition take the new revision; a missing pod below the
 *      partition is recreated at the old one);
 *   3. stop at the first apply that changes no slot and no row field, or after the cycle cap
 *      min(2*C + 8, LWSE_LWS_FORECAST_MAX_CYCLES), or when n' > C (possible only with a negative
 *      maxUnavailable): the replay is then UNFINISHED.
 * Spec edits during the replay are not modelled.  The pass of the current rows runs first; an object
 * whose pass reports LWSE_LOUT_RUP_ERROR, _STATUS_ERROR or _IRREGULAR, or whose C exceeds
 * LWSE_LWS_FORECAST_MAX_SLOTS, runs no cycle (LWSE_LWSF_NOT_FORECAST); one with LWSE_LOUT_BAD_TABLE
 * gets LWSE_LWSF_BAD_TABLE.  Both leave every other field 0 except step_base, which holds the running
 * offset like every object's (such an object has no rows). */
#define LWSE_LWS_FORECAST_MAX_CYCLES 65536u
#define LWSE_LWS_FORECAST_MAX_SLOTS (1u << 20)

typedef struct lwse_lws_forecast { /* per LWS, 32 B */
  uint32_t flags;            /* LWSE_LWSF_* */
  uint32_t cycles;           /* cycles whose apply changed something (= n_steps)                      */
  uint32_t step_base;        /* first trajectory row of this object: rows of the objects before it, in
                                row order (saturates at 0xFFFFFFFF)                                    */
  uint32_t n_steps;          /* trajectory rows of this object                                         */
  int32_t peak_sts_replicas; /* max of the StatefulSet's replicas now (0 without one) and every n'     */
  int32_t floor_ready;       /* min of the ready count now (the pass of the current rows) and, for each
                                cycle, the slots idx < n' that are COUNTED and COND_READY and are not
                                being replaced (idx >= p' without COND_UPDATED) before its apply       */
  int32_t final_partition;   /* (p', n') of the last pass: what the StatefulSet holds when the replay  */
  int32_t final_replicas;    /* stopped, what the controller writes next when it did not               */
} lwse_lws_forecast;

#define LWSE_LWSF_ROLLING (1u << 0)      /* the pass of the current rows is UpdateInProgress            */
#define LWSE_LWSF_WAITING (1u << 1)      /* the first cycle assumes groups that are not ready now become
                                            ready: its apply set STATE_READY or COND_READY on a slot    */
#define LWSE_LWSF_DONE (1u << 2)         /* stopped, and the last pass has LWSE_LOUT_UPDATE_DONE        */
#define LWSE_LWSF_UNFINISHED (1u << 3)   /* stopped by the cycle cap or by n' > C                       */
#define LWSE_LWSF_TRUNCATED (1u << 4)    /* its trajectory did not fit in step_capacity: none of its
                                            rows were written (the summary is exact)                    */
#define LWSE_LWSF_HELD (1u << 5)         /* stopped with final_partition > 0 equal to the spec's
                                            rollingUpdateConfiguration.partition (the clamp :285-288)   */
#define LWSE_LWSF_BAD_TABLE (1u << 6)    /* as LWSE_LOUT_BAD_TABLE                                      */
#define LWSE_LWSF_NOT_FORECAST (1u << 7) /* see above                                                   */

/* One trajectory row: the pass after a cycle whose apply changed something (16 B).  An object's
 * n_steps rows are contiguous at step_base, in cycle order; the last one is the state the replay
 * stopped in (for a stopped replay). */
typedef struct lwse_lws_forecast_step {
  int32_t partition;
  int32_t sts_replicas;
  int32_t ready_replicas;
  int32_t updated_replicas;
} lwse_lws_forecast_step;

/* An object whose rows do not all fit below step_capacity gets LWSE_LWSF_TRUNCATED and writes none;
 * no row at or beyond step_capacity is written, and no object writes outside its own n_steps rows. */
typedef struct lwse_lws_forecast_out {
  lwse_lws_forecast* lws;           /* [n_lws]                                                */
  lwse_lws_forecast_step* steps;    /* [step_capacity], or NULL: summaries only               */
  uint32_t step_capacity;
  uint32_t n_steps_written;         /* out: trajectory rows written                           */
  uint64_t n_steps_needed;          /* out: rows every object's trajectory needs              */
} lwse_lws_forecast_out;

/* Stateless: n_lws object rows and the n_groups group result rows of a sweep of the same tables
 * (only the low five flag bits are read), host memory.  LWSE_ERR_INVALID_ARG for NULL or misaligned
 * tables or outputs; LWSE_ERR_UNSUPPORTED when the objects' slots (C rounded up to 8, summed) reach 2^31.
 * The kernels check every access to their private slots and to the trajectory rows against the sizes
 * the scans gave; an access they refuse would be an engine defect, and fails the call with LWSE_ERR_CUDA
 * and lwse_last_cuda_error() == cudaErrorAssert (710). */
LWSE_API int lwse_lws_forecast_host(lwse_engine* e, const lwse_lws_rec* lws, uint32_t n_lws,
                                    const lwse_group_out* group_out, uint32_t n_groups, lwse_lws_forecast_out* out);
/* Over the resident LWS rows and the resident group results.  The call snapshots both on the engine's
 * stream (device-to-device copies behind the most recently submitted tick, in flight or not) and
 * replays on a stream of its own, with scratch of its own: it never waits for, drains or drops a tick,
 * and touches no tick graph, arena, change list or output.  The scratch only grows (a call that needs
 * more than any before allocates, which waits for the device as cudaMalloc does).  LWSE_ERR_NOT_READY
 * before lwse_resident_load, and while the group results do not belong to the resident rows: after a
 * load, and after a patch of LWS, group or pod rows made without a sweep (lwse_resident_patch, or a
 * tick with LWSE_TICK_NO_SWEEP), until the next sweep is enqueued.  LWSE_ERR_INVALID_ARG for NULL
 * outputs; LWSE_ERR_UNSUPPORTED and LWSE_ERR_CUDA as for lwse_lws_forecast_host. */
LWSE_API int lwse_resident_forecast(lwse_engine* e, lwse_lws_forecast_out* out);

/* ---- rollout what-if ------------------------------------------------------------------------
 * What a proposed edit of a LeaderWorkerSet would make the controller do, before the edit reaches the
 * API server.  A query is a list of proposals (row L_i, lwse_lws_rec P_i), i = 0 .. n-1, each answered on
 * its own as if it were the only edit; several proposals may name the same row (to compare settings).
 *   - Ranges: P_i's group_base and group_count are ignored and taken from the resident row L_i (a
 *     what-if moves no group rows).  Every other field is the caller's: rev_hash, flags (LWSE_LWS_UPDATED,
 *     the percent, restart, startup and exclusive bits, INTSTR_INVALID, IRREGULAR), replicas, partition,
 *     max_surge, max_unavailable, size, subgroup_size and the sts_* fields.  A template edit is rev_hash
 *     set to the new revision's hash plus LWSE_LWS_UPDATED (what the encoder writes for
 *     leaderWorkerSetUpdated, leaderworkerset_controller.go:150-159, :325-332); a scale is a changed
 *     replicas, which Case 4 (:351-361) compares with the annotation the row already carries.
 *   - now[i]: the lwse_lws_out row of L_i in a sweep of the resident tables with row L_i replaced by the
 *     proposal, under the flags of the most recently submitted sweep: what the controller writes first.
 *   - fc.lws[i] and the trajectory: lwse_resident_forecast's row of L_i over the same replaced tables (the
 *     same rules, cap, flags and fields).  Proposal i's trajectory rows are contiguous at step_base; the
 *     offsets run over the proposals in query order, with the TRUNCATED / step_capacity /
 *     n_steps_written / n_steps_needed contract of lwse_lws_forecast_out.
 *   - A group row inside L_i's range whose lws_index is not L_i keeps the result the resident sweep gave
 *     it (its owner and pods are unchanged), so the answer is exactly the full replaced-table sweep's; only
 *     the range rows L_i owns are recomputed.
 *   - A resident row whose range lies outside the group table gets LWSE_LOUT_BAD_TABLE /
 *     LWSE_LWSF_BAD_TABLE, as the sweep and the forecast give it, and gathers no group rows.
 * Readiness, isolation and scratch as lwse_resident_forecast: LWSE_ERR_NOT_READY before
 * lwse_resident_load and while the group results do not belong to the resident rows; the call holds the
 * engine mutex, runs on a stream of its own behind an event on the engine's stream (it sees the most
 * recently submitted tick, in flight or not), reads the resident tables in place, and never waits for,
 * drains or drops a tick or touches a graph, arena, change list, output, occupancy counter, node index or
 * tick info.  LWSE_ERR_INVALID_ARG for NULL or misaligned arrays or a row >= n_lws.  LWSE_ERR_UNSUPPORTED
 * when the proposals' slots reach 2^31 (as the forecast refuses), or when the gathered group rows (the
 * named rows' group_count summed over the proposals whose range lies inside the table) reach 2^32; an
 * unsupported call writes nothing.  n == 0 is a valid empty answer. */
typedef struct lwse_rollout_whatif {
  const uint32_t* rows;      /* [n] resident LWS rows                                */
  const lwse_lws_rec* recs;  /* [n] proposed rows, 16-byte aligned                   */
  uint32_t n;
  uint32_t reserved;
  lwse_lws_out* now;         /* [n] out                                              */
  lwse_lws_forecast_out fc;  /* fc.lws [n]; fc.steps [step_capacity] or NULL          */
} lwse_rollout_whatif;
LWSE_API int lwse_resident_rollout_whatif(lwse_engine* e, lwse_rollout_whatif* q);

/* ------------------------------------------------------------------------- */
/* Placement (build-defined spec — the reference has no node scoring)        */
/* ------------------------------------------------------------------------- */

/* One placement request per pod group of an exclusive-topology object (32 B). */
typedef struct lwse_place_req {
  uint64_t priority;    /* total order: smaller wins (uid_hash-derived)          */
  uint64_t group_key;   /* first 8 bytes of the SHA-1 group key: preference salt */
  uint32_t group;       /* caller's group id, echoed back                        */
  uint32_t ns;          /* dense namespace id: exclusivity is per namespace      */
  int32_t size;         /* pods that must fit in the domain                      */
  uint32_t leader_node; /* node row if the leader is scheduled, else LWSE_NONE   */
} lwse_place_req;

typedef struct lwse_place_out {
  uint32_t domain_id;   /* claimed domain or LWSE_NONE                           */
  uint32_t leader_node; /* chosen (or given) node for the leader, or LWSE_NONE   */
  uint32_t flags;       /* LWSE_PLACE_* */
  uint32_t score;       /* score of the winning (group, node) pair               */
} lwse_place_out;

#define LWSE_PLACE_PLACED (1u << 0)
#define LWSE_PLACE_PINNED (1u << 1)        /* domain came from a scheduled leader */
#define LWSE_PLACE_CONFLICT (1u << 2)      /* pinned domain already held by a
                                              higher-priority group              */
#define LWSE_PLACE_UNSCHEDULABLE (1u << 3) /* no feasible domain left            */

/* occupancy: pods per node (n_nodes counters, host memory) already summed over
 * every shard; NULL = all zero. */
LWSE_API int lwse_place_host(lwse_engine* e, const lwse_place_req* reqs, uint32_t n_reqs,
                             const uint32_t* occupancy, uint32_t n_namespaces,
                             lwse_place_out* out, uint32_t* rounds_out);
/* Device pointers; enqueued on `stream`.  rounds_out == NULL: no synchronize;
 * otherwise the call waits for the round count.  The placement rounds of one engine share
 * its scratch: they must not overlap in time — keep them on one stream (lwse_reconcile_*
 * use the engine's side stream for theirs) or order the streams with events. */
LWSE_API int lwse_place_device(lwse_engine* e, const lwse_place_req* d_reqs, uint32_t n_reqs,
                               const uint32_t* d_occupancy, uint32_t n_namespaces,
                               lwse_place_out* d_out, uint32_t* rounds_out, void* stream);

/* As lwse_place_device for a request table the caller keeps GROUPED BY NAMESPACE (ns
 * non-decreasing): one CTA per namespace, holder table / capacities / node table in shared memory
 * (the latter staged by TMA).  flags: LWSE_SWEEP_PLACE_SCAN.  pair_scans_out (optional, with
 * rounds_out): number of (request, round) searches the call made — x usable nodes = (request x
 * node) pairs the scan form scored. */
LWSE_API int lwse_place_grouped_device(lwse_engine* e, const lwse_place_req* d_reqs, uint32_t n_reqs,
                                       const uint32_t* d_occupancy, uint32_t n_namespaces, lwse_place_out* d_out,
                                       uint32_t flags, uint32_t* rounds_out, uint32_t* pair_scans_out, void* stream);

/* Multi-GPU form: `d_parts` is the result of ONE all-gather over the ranks; part p
 * (rank p, at d_parts + p * part_stride_bytes) holds that shard's per-node occupancy
 * (n_nodes uint32 counters) followed, at reqs_offset_bytes, by reqs_per_part request
 * rows (unused rows: leader_node = LWSE_NONE, size = 0).  Node occupancy is summed over
 * the parts; request r = p * reqs_per_part + j; d_out has n_parts * reqs_per_part rows.
 * Every rank solves the same problem and keeps the rows of its own part. */
LWSE_API int lwse_place_gathered_device(lwse_engine* e, const void* d_parts, uint32_t n_parts,
                                        uint64_t part_stride_bytes, uint64_t reqs_offset_bytes,
                                        uint32_t reqs_per_part, uint32_t n_namespaces,
                                        lwse_place_out* d_out, uint32_t* rounds_out, void* stream);

/* One reconcile tick on device tables: lwse_sweep_lws_device(d) on `stream` and a
 * placement round (as lwse_place_device, rounds_out = NULL) on an engine-owned side
 * stream, forked from and joined back into `stream` with events — the placement
 * round reads only its own inputs, never the sweep's outputs, so the two overlap.
 * This is what one pass of the controller's work queue maps to: every
 * Reconcile() (leaderworkerset_controller.go:106-193, pod_controller.go:71-201)
 * plus the scheduler's share of the exclusive-topology contract.
 * n_reqs == 0: sweep only. */
LWSE_API int lwse_reconcile_device(lwse_engine* e, const lwse_lws_tables* d, const lwse_place_req* d_reqs,
                                   uint32_t n_reqs, const uint32_t* d_occupancy, uint32_t n_namespaces,
                                   lwse_place_out* d_place_out, void* stream);

/* The same tick from host tables: lwse_sweep_lws_host(host) and lwse_place_host(reqs, …) in one
 * call, the placement round solved on the side stream while the sweep's tables are uploaded;
 * returns when all results are in the caller's buffers.  n_reqs == 0: sweep only.
 * host->flags & LWSE_SWEEP_PLACE_GROUPED: the request table is grouped by namespace — the call then
 * skips its own pass over the table (it is checked on the device instead: LWSE_ERR_BAD_TABLE when
 * the promise does not hold; without the flag the call finds out itself). */
LWSE_API int lwse_reconcile_host(lwse_engine* e, const lwse_lws_tables* host, const lwse_place_req* reqs,
                                 uint32_t n_reqs, const uint32_t* occupancy, uint32_t n_namespaces,
                                 lwse_place_out* place_out);

/* ---- placement what-if -----------------------------------------------------------------------
 * "If these nodes were cordoned / relabelled / resized, or these requests changed or were added, what
 * would the placement round give?" — answered on the resident tables without changing them.
 *
 * The what-if round is the round the placement spec computes over: the resident node rows with the
 * NODES patches applied, the resident occupancy counters, the resident request rows with the PLACE_REQS
 * patches applied followed by the `extra` rows, and n_namespaces namespaces.  Requests with
 * ns >= n_namespaces get the tick's UNSCHEDULABLE row; extra row i has row index (and key) rn_reqs + i,
 * where rn_reqs is the resident request count.  Identity patches are not taken: node deletion and
 * eviction move occupancy, which a what-if never does.
 *
 * The baseline ("before") is the rows of the most recently submitted tick that ran LWSE_TICK_PLACE, in
 * flight or not.  For a query without extra rows and with the resident n_namespaces, `after` equals byte
 * for byte the rows a tick with the same segments and LWSE_TICK_PLACE computes, and {rows} is that
 * tick's place change list.
 *
 * Namespaces are independent sub-problems over one capacity snapshot: without node patches the call
 * solves only the TOUCHED namespaces (old and new namespace of every patched request row, the namespace
 * of every extra row, and the namespaces n_namespaces adds) and every other row keeps its baseline row;
 * with node patches it solves every namespace.  Node patches that change a node's usability or the
 * domain of a usable node (the tick's rule) build a what-if node index; others use the resident one.
 *
 * Isolation: the call runs under the engine mutex, on a stream of its own with scratch of its own,
 * behind everything the engine's stream holds (the most recently submitted tick with both branches
 * joined).  It never drains, waits for the results of, or drops a tick, and touches no tick graph,
 * arena region, change list, resident table, node index, output row, occupancy counter or tick info.
 * Its segments are copied into a pinned staging buffer of its own.  Its scratch only grows (a call that
 * needs more than any before allocates, which waits for the device as cudaMalloc does).
 *
 * Returns LWSE_ERR_NOT_READY before lwse_resident_place_load, before the first tick with
 * LWSE_TICK_PLACE, and while the rows of that tick do not belong to the resident tables: after node,
 * request or identity rows were patched by a tick without LWSE_TICK_PLACE, by lwse_resident_patch, or
 * replaced by lwse_upload_nodes / lwse_resident_load, until the next tick with it.  An empty resident
 * request table is ready after such a tick too (its baseline is empty): a what-if with extra rows only
 * is the admission check of the first exclusive object.  LWSE_ERR_INVALID_ARG for a NULL
 * query, more than LWSE_TICK_MAX_SEGS segments, a table other than LWSE_TABLE_NODES or
 * LWSE_TABLE_PLACE_REQS, a scattered row at or beyond its table, n_namespaces == 0 with no resident
 * count, or a NULL buffer with a count > 0; LWSE_ERR_BAD_TABLE for a range segment beyond its table (as
 * a tick).  LWSE_ERR_UNSUPPORTED when rn_reqs + n_extra >= 2^24 (row keys are 24-bit) and on an
 * engine with a peer exchange (the shared-occupancy round).  The scan form is not offered (it gives
 * the same rows by spec); where a tick would run the general form (the domains do not fit one CTA) the
 * what-if does too. */
typedef struct lwse_place_whatif {
  /* in */
  const lwse_patch_seg* segs;     /* LWSE_TABLE_NODES and LWSE_TABLE_PLACE_REQS only, the packing of a
                                     tick's segments, host memory                                      */
  uint32_t n_segs;
  const lwse_place_req* extra;    /* hypothetical new requests: rows rn_reqs .. rn_reqs + n_extra - 1   */
  uint32_t n_extra;
  uint32_t n_namespaces;          /* 0 = the resident count; may be larger (new namespaces)            */
  uint32_t capacity;              /* rows the change buffers below hold                                */
  uint32_t* rows;                 /* [capacity]: resident rows whose row differs from the baseline      */
  lwse_place_out* before;         /* [capacity]: their baseline rows                                    */
  lwse_place_out* after;          /* [capacity]: their what-if rows                                     */
  lwse_place_out* extra_out;      /* [n_extra], always written                                          */
  /* out */
  uint32_t n_changed;             /* every resident row that differs (rows beyond capacity not listed;
                                     order unspecified)                                                */
  uint32_t n_lost;                /* PLACED before and not after (resident rows)                       */
  uint32_t n_moved;               /* PLACED in both, in another domain                                  */
  uint32_t n_gained;              /* not PLACED before, PLACED after                                    */
  uint32_t n_placed;              /* PLACED / UNSCHEDULABLE / CONFLICT rows of the whole what-if round, */
  uint32_t n_unschedulable;       /* extra rows included                                                */
  uint32_t n_conflict;
  uint32_t namespaces_solved;     /* namespaces the namespace form solved (0 for the general form)      */
  uint32_t form;                  /* LWSE_TICK_FORM_NAMESPACE or LWSE_TICK_FORM_GENERAL                 */
} lwse_place_whatif;
LWSE_API int lwse_resident_place_whatif(lwse_engine* e, lwse_place_whatif* q);

/* ---- placement explanation -------------------------------------------------------------------
 * "Why is this group not placed?" — for each chosen row of a placement round, which domains fit it, which are
 * held ahead of it in its namespace and by whom, and by how many free slots it falls short.  The answer
 * describes the given round; it is not itself a what-if.
 *
 * The round.  Without segments, without extra rows and with n_namespaces 0 or the resident count, the round
 * explained is the BASELINE: the rows of the most recently submitted tick with LWSE_TICK_PLACE (in flight or
 * not), over the resident node rows, occupancy counters and request rows.  Otherwise it is the WHAT-IF round
 * lwse_resident_place_whatif computes for the same segs, extra and n_namespaces (the same meaning and the same
 * refusals; extra row i is row rn_reqs + i).  A what-if with none of them gives the baseline's rows, so the two
 * agree where they meet.  Rollout placement is defined as such a what-if, so explaining an entry's E_i as extra
 * rows explains exactly the rows that entry strands.
 *
 * The rows.  With `rows` non-NULL, the n_rows listed row indices into the round, in the given order (duplicates
 * allowed); with `rows` NULL, every row of the round whose lwse_place_out flags share a bit with `mask`, in
 * ascending row order.  The first `capacity` are written to `out`; n_explained counts them all, and the totals
 * cover them all.
 *
 * Per domain d of the round (n_domains of the node table), over the round's node rows and the resident
 * occupancy occ[n]:
 *   dom_free[d]  the spec's Σ free[n] (DESIGN.md §7: schedulable, labelled nodes of d, max(0, capacity − occ));
 *   usable[d]    the number of schedulable labelled nodes of d;
 *   free_all[d]  Σ max(0, capacity − occ) over every node labelled into d, schedulable or not (uint32), i.e.
 *                dom_free[d] with the cordons lifted.
 * The holder of (ns, d) is the PLACED row of the round, pinned or not, whose namespace is ns and domain is d;
 * its key is the spec's key (the low 24 bits are its row).  A round has at most one.
 *
 * Explained row r, with spec key k, namespace ns < n_namespaces and size s (compared as signed integers): each
 * domain falls in exactly one class, tested in this order:
 *   own           r is PLACED in d;
 *   no_usable     usable[d] == 0;
 *   too_small     dom_free[d] < s;
 *   held_pinned   (d fits) held by a pinned row with key < k;
 *   held_earlier  (d fits) held by an unpinned row with key < k;
 *   held_later    (d fits) held by a row with key > k;
 *   open          (d fits) not held.
 * fit_uncordoned counts the no_usable and too_small domains with free_all[d] >= s.  Named domains (LWSE_NONE
 * when the set is empty):
 *   best_domain      the argmax of the spec's level-1 hash hi = mix(key_lo ^ d·φ) | 1 over own, held_later and
 *                    open, ties to the lower d: the domain the serial order gives an unpinned r;
 *   blocker_domain   the argmax of hi over held_pinned and held_earlier, ties to the lower d, and blocker_row its
 *                    holder: the domain r would take if that holder were gone;
 *   shortfall_domain the too_small domain with the smallest s − dom_free[d] (= shortfall), ties to the lower d:
 *                    the free slots r lacks in the closest domain too small for it.
 * Row flags (LWSE_PEX_*): CAPACITY, no domain fits (usable[d] > 0 and dom_free[d] >= s); EXCLUSIVE, some fit and
 * every one is held ahead of r; CORDONED, fit_uncordoned > 0 (a domain would fit with its cordoned nodes
 * counted — not that r would place: lwse_resident_place_whatif with uncordoning segments answers that);
 * CONFLICT, r is pinned and its leader's domain is held by a smaller pinned key (blocker_domain / blocker_row
 * are then that domain and its holder); NO_CLAIM, r is pinned and its leader's node is missing, unlabelled or
 * out of range; BAD_SIZE, r is unpinned with s < 1.  CAPACITY, EXCLUSIVE and CORDONED describe the domains as
 * an unpinned request of r's size and key would see them; a pinned row's domain comes from its leader.  A row
 * with ns >= n_namespaces carries NO_NAMESPACE alone: no domain is classified and every count is 0.
 *
 * The certificate.  The spec serves unpinned requests in ascending key order (a serial dictatorship), so in any
 * round an UNSCHEDULABLE unpinned row of size >= 1 has open + held_later == 0, and a PLACED unpinned row has
 * best_domain == its domain_id and score == hi(best_domain).
 *
 * Readiness, errors and isolation: exactly lwse_resident_place_whatif's — LWSE_ERR_NOT_READY and
 * LWSE_ERR_UNSUPPORTED as it returns them (a peer exchange; rn_reqs + n_extra >= 2^24), the same
 * LWSE_ERR_INVALID_ARG for segments, extra rows and namespaces, and LWSE_ERR_INVALID_ARG for a listed row at or
 * beyond the round's row count or a NULL buffer with a count > 0.  A refused call writes nothing.  The call
 * holds the engine mutex, runs on the what-if stream behind an event on the engine's stream, uses the what-if's
 * scratch for a what-if round and scratch of its own (which only grows) for the explanation, and touches
 * nothing of a tick.  Where the what-if runs the general form, so does the explained round. */
typedef struct lwse_place_explain_row {
  uint32_t row;              /* row of the round                                                        */
  uint32_t flags;            /* LWSE_PEX_*                                                              */
  uint32_t place_flags;      /* the round's lwse_place_out flags of the row                             */
  uint32_t n_own;            /* the classes above: they sum to n_domains (0 with LWSE_PEX_NO_NAMESPACE) */
  uint32_t n_no_usable;
  uint32_t n_too_small;
  uint32_t n_held_pinned;
  uint32_t n_held_earlier;
  uint32_t n_held_later;
  uint32_t n_open;
  uint32_t n_fit_uncordoned;
  uint32_t best_domain;
  uint32_t blocker_domain;
  uint32_t blocker_row;
  uint32_t shortfall;        /* 0 when shortfall_domain is LWSE_NONE                                    */
  uint32_t shortfall_domain;
} lwse_place_explain_row;   /* 64 B */

#define LWSE_PEX_CAPACITY (1u << 0)
#define LWSE_PEX_EXCLUSIVE (1u << 1)
#define LWSE_PEX_CORDONED (1u << 2)
#define LWSE_PEX_CONFLICT (1u << 3)
#define LWSE_PEX_NO_CLAIM (1u << 4)
#define LWSE_PEX_NO_NAMESPACE (1u << 5)
#define LWSE_PEX_BAD_SIZE (1u << 6)

typedef struct lwse_place_explain_query {
  /* in: the round (as lwse_place_whatif) */
  const lwse_patch_seg* segs;
  uint32_t n_segs;
  uint32_t n_extra;
  const lwse_place_req* extra;
  uint32_t n_namespaces;
  /* in: the rows */
  uint32_t mask;                    /* with rows == NULL: LWSE_PLACE_* bits that select a row               */
  const uint32_t* rows;             /* [n_rows] row indices into the round, host memory; NULL: by mask      */
  uint32_t n_rows;
  uint32_t capacity;                /* rows `out` holds                                                     */
  lwse_place_explain_row* out;      /* [capacity], host memory                                              */
  /* out */
  uint32_t n_explained;             /* rows selected (beyond capacity counted, not written)                 */
  uint32_t round_rows;              /* rows of the round (rn_reqs + n_extra)                                */
  uint32_t n_domains;
  uint32_t whatif;                  /* 1: the what-if round was explained, 0: the baseline                   */
  uint32_t form;                    /* the what-if's form (LWSE_TICK_FORM_*), 0 for the baseline             */
  uint32_t n_flag[7];               /* rows carrying LWSE_PEX_* bit i                                        */
  uint64_t n_class[8];              /* sums over the rows of n_own .. n_fit_uncordoned                       */
} lwse_place_explain_query;
LWSE_API int lwse_resident_place_explain(lwse_engine* e, lwse_place_explain_query* q);

/* ---- drain what-if ------------------------------------------------------------------------------
 * "If I drain these nodes, which LeaderWorkerSet groups restart?" — answered on the resident tables
 * without changing them.  With RecreateGroupOnPodRestart / RecreateGroupAfterStart, evicting one pod of
 * a group deletes its leader and so recreates the whole group (handleRestartPolicy,
 * pod_controller.go:204-266, behind the pending gate of pendingPodsInGroup :338-362 and the owner chain
 * of workerPodBelongsToLeader :268-295).
 *
 * Definition: for a set D of node rows, the what-if rows are the group result rows of a sweep of the
 * resident tables (the sweep flags of the most recently submitted sweep) with two changes — the rows the
 * informer produces when eviction sets deletionTimestamp on every pod bound to those nodes:
 *   - LWSE_POD_DELETING is set in the state byte of every pod whose identity row has LWSE_PODID_SCHEDULED
 *     and a node field in D;
 *   - LWSE_GRP_POD_DELETING is set on every group row whose leader_node is in D.
 * Nothing else changes.  The LWS pass reads only the five low flag bits of a group result row, which
 * eviction changes on no row, so the LWS result rows do not change and only group rows are returned.
 *
 * The baseline ("before") is the group results of the most recently submitted sweep, in flight or not:
 * the rows lwse_resident_forecast snapshots, under the same readiness rule.
 *
 * Isolation: as lwse_resident_place_whatif — under the engine mutex, on the what-if stream behind an event
 * recorded on the engine's stream, with scratch of its own (a copy of the pod-state column and of the
 * group rows, the sweep's bitmaps and result rows); it never drains, waits for the results of, or drops a
 * tick, and touches no tick graph, arena, change list, resident table, output row, occupancy counter, node
 * index or tick info.  The scratch only grows.
 *
 * Multi-rank engines: both calls see only this rank's objects.  Every count is a sum over groups and a
 * group lives on one rank, so the sum of the ranks' answers is the cluster's answer.
 *
 * Returns LWSE_ERR_NOT_READY before lwse_resident_load, before a node table is uploaded, and while the
 * group results do not belong to the resident rows (after a load, and after a patch of LWS, group or pod
 * rows made without a sweep, until the next sweep is enqueued).  LWSE_ERR_INVALID_ARG for a NULL query, a
 * node row at or beyond n_nodes, or a NULL buffer with a count > 0.  Duplicate node rows are allowed. */
typedef struct lwse_drain_whatif {
  /* in */
  const uint32_t* nodes;      /* [n_nodes] node rows of D, host memory                                  */
  uint32_t n_nodes;
  uint32_t capacity;          /* rows the change buffers below hold                                     */
  uint32_t* rows;             /* [capacity]: group rows whose result differs from the baseline          */
  lwse_group_out* before;     /* [capacity]: their baseline rows                                        */
  lwse_group_out* after;      /* [capacity]: their what-if rows                                         */
  /* out */
  uint32_t n_changed;         /* every group row that differs (rows beyond capacity not listed; order
                                 unspecified)                                                          */
  uint32_t n_pods_evicted;    /* identity rows scheduled on a node of D                                 */
  uint32_t n_leaders_evicted; /* group rows whose leader_node is in D                                   */
  uint32_t n_groups_restarted;/* LWSE_GOUT_DELETE_LEADER | LWSE_GOUT_LEADER_DELETING clear before, set
                                 after                                                                 */
  uint32_t n_ready_restarted; /* of those, the groups with LWSE_GOUT_COND_READY in the baseline         */
  uint32_t reserved;
  uint64_t n_pods_recreated;  /* sum of pod_count over the restarted groups                             */
} lwse_drain_whatif;
LWSE_API int lwse_resident_drain_whatif(lwse_engine* e, lwse_drain_whatif* q);

/* The drain cost of every node of the resident node table: row n holds the totals of
 * lwse_resident_drain_whatif with D = {n}, all nodes in one pass (32 B per node).  Exact in one pass: take
 * a group whose baseline has neither restart bit.  Draining n restarts it iff some pod of the group bound
 * to n passes handleRestartPolicy with its deleting bit set; that per-pod verdict reads only the pod's
 * state byte and identity row, the group row and the group's pending state (none of which the deletion of
 * other pods changes), and the leader's deleting bit only chooses between DELETE_LEADER and
 * LEADER_DELETING.  A group that already has a restart bit never counts.  Same readiness, isolation and
 * errors as lwse_resident_drain_whatif; `out` holds n_nodes rows of host memory. */
typedef struct lwse_drain_cost {
  uint32_t pods;             /* n_pods_evicted = lwse_resident_occupancy[n]                             */
  uint32_t leaders;          /* n_leaders_evicted                                                       */
  uint32_t groups_restarted; /* n_groups_restarted                                                      */
  uint32_t ready_restarted;  /* n_ready_restarted                                                       */
  uint64_t pods_recreated;   /* n_pods_recreated                                                        */
  uint64_t reserved;
} lwse_drain_cost;
LWSE_API int lwse_resident_drain_cost(lwse_engine* e, lwse_drain_cost* out);

/* ---- drain budget -------------------------------------------------------------------------------
 * "Does this drain take a LeaderWorkerSet below its availability floor?"  LeaderWorkerSet has no
 * disruption budget of its own; the one number that says how many groups an object may lose is
 * rollingUpdateConfiguration.maxUnavailable, which the controller respects on rolling updates
 * (leaderworkerset_controller.go:302, :366-369, :650-673).  The reference has no drain budget: the
 * definition below is this build's own (DESIGN.md §3.5, "Drain budget").
 *
 * Definition.  An LWS row L is EVALUATED when its baseline result row has none of LWSE_LOUT_BAD_TABLE,
 * _IRREGULAR, _RUP_ERROR, _STATUS_ERROR and its row has no LWSE_LWS_INTSTR_INVALID.  For an evaluated L:
 *   floor        = max(0, replicas - mu), mu = maxUnavailable scaled against replicas, rounded down (:302),
 *                  in 64 bits as Go's int (mu is never truncated to int32); the floor is clamped to int32;
 *   ready_before = lws_out[L].ready_replicas of the baseline (the results of the most recently submitted
 *                  sweep, the rows lwse_resident_drain_whatif diffs against).
 * The groups of L are the rows g of its group range (inside the group table) with lws_index == L.  For a
 * drain set D of node rows a group is RESTARTED exactly as lwse_resident_drain_whatif defines it (neither
 * restart bit in its baseline row, one in its what-if row), and
 *   lost         = restarted groups of L whose baseline row has LWSE_GOUT_COND_READY (counted into
 *                  readyReplicas, :455-458);  ready_after = ready_before - lost;
 *   BREACHED        lost > 0 and ready_after < floor;
 *   ALREADY_BELOW   ready_before < floor, whether or not D touches L;
 *   LOSES_AVAILABLE the baseline condition is Available and a lost group has index g - group_base <
 *                   replicas (readyNonBurstWorkerCount falls below replicas, :494).
 * L is TOUCHED when any group of L restarts.  A touched L that is not evaluated is listed with
 * LWSE_DRAINB_NOT_EVALUATED (floor 0) and counts in n_touched / lws_touched only.
 *
 * Drain sets: LWSE_DRAIN_NODES takes node rows (as lwse_resident_drain_whatif); LWSE_DRAIN_DOMAINS takes
 * domain ids below the resident n_domains and drains every node row whose domain_id is one of them — by
 * domain_id alone, so cordoned and unschedulable nodes belong to their domain, and a node whose domain_id
 * is LWSE_NONE or >= n_domains belongs to none.
 *
 * Readiness, isolation and errors: as lwse_resident_drain_whatif (the what-if stream, the engine mutex,
 * scratch of its own that only grows; no tick, graph, arena, change list, resident table, output row,
 * occupancy counter, node index or tick info is touched).  LWSE_ERR_INVALID_ARG also for a scope other
 * than the two, and for a domain id >= n_domains.  Multi-rank engines: an LWS lives on one rank, so every
 * count sums across ranks' answers and min_margin is the min of theirs. */
#define LWSE_DRAIN_NODES 0u
#define LWSE_DRAIN_DOMAINS 1u

#define LWSE_DRAINB_NOT_EVALUATED (1u << 0)
#define LWSE_DRAINB_BREACHED (1u << 1)
#define LWSE_DRAINB_ALREADY_BELOW (1u << 2)
#define LWSE_DRAINB_LOSES_AVAILABLE (1u << 3)

/* One touched LWS row of a drain (32 B). */
typedef struct lwse_drain_budget {
  uint32_t lws;               /* LWS row                                                                */
  uint32_t flags;             /* LWSE_DRAINB_*                                                           */
  int32_t replicas;           /* spec.replicas                                                           */
  int32_t floor;              /* 0 when not evaluated                                                    */
  int32_t ready_before;
  int32_t ready_after;        /* ready_before - lost, clamped to int32                                   */
  uint32_t groups_restarted;  /* restarted groups of L, ready or not                                     */
  uint32_t reserved;
} lwse_drain_budget;

/* The set form: the touched LWS rows of one drain set, and its totals. */
typedef struct lwse_drain_budget_query {
  /* in */
  const uint32_t* ids;        /* [n_ids] node rows or domain ids (by scope), host memory; duplicates allowed */
  uint32_t n_ids;
  uint32_t scope;             /* LWSE_DRAIN_NODES or LWSE_DRAIN_DOMAINS                                  */
  uint32_t capacity;          /* rows `rows` holds                                                       */
  uint32_t reserved;
  lwse_drain_budget* rows;    /* [capacity]: touched LWS rows (beyond capacity not listed; order unspecified) */
  /* out */
  uint32_t n_touched;         /* every touched LWS row, listed or not                                    */
  uint32_t n_breached;
  uint32_t n_loses_available;
  uint32_t n_already_below;   /* evaluated rows below their floor, touched or not                       */
  uint32_t n_pods_evicted;    /* the five totals of lwse_drain_whatif for the same node set              */
  uint32_t n_leaders_evicted;
  uint32_t n_groups_restarted;
  uint32_t n_ready_restarted;
  uint64_t n_pods_recreated;
} lwse_drain_budget_query;
LWSE_API int lwse_resident_drain_budget(lwse_engine* e, lwse_drain_budget_query* q);

/* The per-key form: one row per node (LWSE_DRAIN_NODES, n_nodes rows) or per domain (LWSE_DRAIN_DOMAINS,
 * n_domains rows), row k holding the answer of the set form for the node k or for the nodes of domain k
 * (48 B).  The first 32 bytes are an lwse_drain_cost row: for scope NODES they equal
 * lwse_resident_drain_cost byte for byte.  Exact in one pass per key by the drain cost's argument: draining
 * D restarts a group iff some pod of the group bound to a node of D passes the restart verdict with its
 * deleting bit set, so lost(L, key) is the number of distinct COND_READY groups of L with such a pod on the
 * key.  The (LWS, key) pairs are gathered in an open-addressing table in scratch sized from a counting pass
 * (one host synchronisation); an insert the table refuses fails the call with LWSE_ERR_OOM.  `out` holds the
 * rows in host memory. */
typedef struct lwse_drain_budget_cost {
  uint32_t pods;              /* the lwse_drain_cost totals of the key                                   */
  uint32_t leaders;
  uint32_t groups_restarted;
  uint32_t ready_restarted;
  uint64_t pods_recreated;
  uint64_t reserved;
  uint32_t lws_touched;       /* n_touched of the set form for this key                                  */
  uint32_t lws_breached;
  uint32_t lws_loses_available;
  int32_t min_margin;         /* min over touched evaluated L of ready_after - floor; INT32_MAX for none */
} lwse_drain_budget_cost;
LWSE_API int lwse_resident_drain_budget_cost(lwse_engine* e, uint32_t scope, lwse_drain_budget_cost* out);

/* ---- drain waves --------------------------------------------------------------------------------
 * "Which of these nodes (domains) can I drain together?"  A first-fit plan of a list of keys into waves whose
 * set-form drain budget breaches no LeaderWorkerSet (DESIGN.md §3.5, "Drain waves").
 *
 * Definition.  ids[0..n_ids) are DISTINCT node rows (LWSE_DRAIN_NODES) or domain ids (LWSE_DRAIN_DOMAINS);
 * scope, drain sets, EVALUATED, floor, ready_before, lost(L, D) and BREACHED are those of
 * lwse_resident_drain_budget.  Waves W_0, W_1, ... start empty; the keys are taken in the caller's order and
 * key k_i gets the first of:
 *   1. LWSE_DRAINW_BREACHES_ALONE  the set form over {k_i} has n_breached > 0 (wave LWSE_NONE);
 *   2. LWSE_DRAINW_PLANNED         wave w: the smallest index of an open wave such that the set form over
 *                                  W_w ∪ {k_i} has n_breached == 0; with no such wave and fewer than max_waves
 *                                  open, a new wave is opened for it;
 *   3. LWSE_DRAINW_NO_WAVE         neither (wave LWSE_NONE).
 * Every wave is judged against the same baseline (the most recently submitted sweep): the plan assumes that
 * the groups one wave restarts are ready again before the next starts, so a controller drains wave 0, waits
 * for recovery and calls again with the keys that remain.  The answer is the first-fit outcome of that
 * sequential order, whatever the device interleaving; first-fit does not promise the fewest waves.
 *
 * Exact through the per-key restart pairs: draining a union of keys restarts the union of the groups each
 * key restarts alone, so lost(L, W) is the number of distinct ready member groups of L among the pairs of W's
 * keys, and adding k to W is admissible iff every evaluated L to which k adds new > 0 such groups has
 * lost(L, W) + new <= ready_before - floor (in 64 bits).
 *
 * Readiness, isolation and errors: as lwse_resident_drain_budget, and LWSE_ERR_INVALID_ARG also for a
 * duplicate or out-of-range id, max_waves of 0 or above LWSE_DRAIN_WAVES_MAX, a NULL ids / keys (n_ids > 0)
 * or waves, or a nonzero reserved field; LWSE_ERR_UNSUPPORTED on an engine with a peer exchange (a plan is not
 * a sum over ranks); LWSE_ERR_OOM rather than a wrong row when a sized scratch table refuses an entry.  A
 * refused call writes no output.  n_ids = 0 is valid and opens no wave. */
#define LWSE_DRAIN_WAVES_MAX 64u

#define LWSE_DRAINW_PLANNED 0u
#define LWSE_DRAINW_BREACHES_ALONE 1u
#define LWSE_DRAINW_NO_WAVE 2u

/* One key of the plan, in query order (32 B).  The alone columns equal row `id` of
 * lwse_resident_drain_budget_cost for the same scope. */
typedef struct lwse_drain_wave_key {
  uint32_t id;                /* the node row or domain id                                               */
  uint32_t wave;              /* its wave, or LWSE_NONE                                                  */
  uint32_t status;            /* LWSE_DRAINW_*                                                           */
  uint32_t groups_restarted;  /* the key alone                                                           */
  uint32_t ready_restarted;
  uint32_t lws_touched;
  uint32_t lws_breached;
  uint32_t reserved;
} lwse_drain_wave_key;

/* One opened wave (48 B): the set-form totals of lwse_resident_drain_budget over the wave's ids. */
typedef struct lwse_drain_wave {
  uint32_t n_keys;
  uint32_t lws_touched;
  uint32_t lws_loses_available;
  uint32_t n_pods_evicted;
  uint32_t n_leaders_evicted;
  uint32_t n_groups_restarted;
  uint32_t n_ready_restarted;
  int32_t min_margin;         /* min over evaluated touched L of ready_after - floor; INT32_MAX for none */
  uint64_t n_pods_recreated;
  uint64_t reserved;
} lwse_drain_wave;

typedef struct lwse_drain_waves_query {
  /* in */
  const uint32_t* ids;        /* [n_ids] distinct node rows or domain ids (by scope), host memory        */
  uint32_t n_ids;
  uint32_t scope;             /* LWSE_DRAIN_NODES or LWSE_DRAIN_DOMAINS                                  */
  uint32_t max_waves;         /* 1 .. LWSE_DRAIN_WAVES_MAX                                               */
  uint32_t reserved;          /* 0                                                                       */
  lwse_drain_wave_key* keys;  /* [n_ids] out                                                             */
  lwse_drain_wave* waves;     /* [max_waves] out: rows 0 .. n_waves                                      */
  /* out */
  uint32_t n_waves;
  uint32_t n_planned;
  uint32_t n_breaches_alone;
  uint32_t n_no_wave;
} lwse_drain_waves_query;
LWSE_API int lwse_resident_drain_waves(lwse_engine* e, lwse_drain_waves_query* q);

/* ---- drain placement ----------------------------------------------------------------------------
 * "If I drain this node or this domain, do the groups it restarts find a new exclusive domain?" — for every
 * node (LWSE_DRAIN_NODES, n_nodes rows) or every domain (LWSE_DRAIN_DOMAINS, n_domains rows) in one call.
 *
 * Definition.  Key k names a node row, or a domain id whose node set is every node row with that domain_id
 * (by domain_id alone, as the drain budget).  Let N_k be that node set.  Row k is the answer of the set-form
 * composition lwse_resident_drain_whatif(N_k) -> unpin -> lwse_resident_place_whatif for D = N_k:
 *   - the restarted groups are those of lwse_resident_drain_whatif(N_k): restart bits clear in the baseline
 *     group results (the most recently submitted sweep), set after;
 *   - U_k, the unpinned requests, are the resident request rows r with leader_node != LWSE_NONE whose
 *     leader_node is in N_k or whose `group` field names a group row below the resident group count that the
 *     drain restarts; the query gives them leader_node = LWSE_NONE;
 *   - the placement is the what-if round (lwse_resident_place_whatif) over the resident node rows with
 *     LWSE_NODE_SCHEDULABLE cleared on N_k, the resident occupancy counters, the resident request rows with
 *     U_k unpinned and the resident n_namespaces, diffed against the rows of the most recently submitted tick
 *     with LWSE_TICK_PLACE.  Occupancy does not move, so the answer is conservative: the pods of a restarted
 *     group on nodes that are not drained still count against those nodes.
 *
 * Locality.  Per key the call solves only the namespaces the key can change, and every other row keeps its
 * baseline row (DESIGN.md §3.5, "Drain placement"): a namespace v is solved for key k when (a) it holds a row
 * of U_k, or (b) it has a row that is not pinned and is PLACED in a drained domain d and either k is a
 * domain, or k is a node n with dom_free[d] - free[n] < size or n the row's chosen node.
 *
 * Readiness and errors: LWSE_ERR_NOT_READY when lwse_resident_drain_whatif or lwse_resident_place_whatif
 * would answer it, or when the resident request table has no namespace; LWSE_ERR_INVALID_ARG for a NULL
 * `out` or another scope; LWSE_ERR_UNSUPPORTED on an engine with a peer exchange, when the resident request
 * count reaches 2^24, and where the namespace form does not fit the domains (the set-form composition then
 * remains the answer); LWSE_ERR_OOM rather than a wrong row when a sized table refuses an entry.
 * Isolation: as the drain what-if (the engine mutex, the what-if stream behind an event on the engine's
 * stream, scratch of its own that only grows; no tick, graph, arena, change list, table, output row,
 * occupancy counter, node index or tick info is touched).  `out` holds the rows in host memory (64 B each). */
typedef struct lwse_drain_place_cost {
  uint32_t groups_restarted;  /* the drain cost's groups_restarted for the key                           */
  uint32_t unpinned;          /* |U_k|                                                                   */
  uint32_t stranded;          /* rows of U_k that are not PLACED after                                   */
  uint32_t bumped;            /* rows outside U_k that are PLACED before and not after                   */
  uint32_t n_changed;         /* the lwse_place_whatif counters of the composed query                    */
  uint32_t n_lost;
  uint32_t n_moved;
  uint32_t n_gained;
  uint32_t n_placed;
  uint32_t n_unschedulable;
  uint32_t n_conflict;
  uint32_t namespaces_solved; /* namespaces the call solved for this key                                 */
  uint32_t reserved[4];
} lwse_drain_place_cost;
LWSE_API int lwse_resident_drain_place_cost(lwse_engine* e, uint32_t scope, lwse_drain_place_cost* out);

/* ---- drain placement waves ----------------------------------------------------------------------
 * "Which of these nodes (domains) can I drain together so that every group the drain restarts finds a new
 * exclusive domain?"  The first-fit plan of lwse_resident_drain_waves with a wave rule that also reads the
 * set-form drain placement (DESIGN.md §3.5, "Drain placement waves").
 *
 * Definition.  ids, scope, max_waves, drain sets, EVALUATED, floor and lost(L, D) are those of
 * lwse_resident_drain_waves.  For a drain set S with node set N_S (the union of its keys' node sets) the
 * placement verdicts come from the set-form composition that lwse_resident_drain_place_cost states for one
 * key, applied to N_S: the groups lwse_resident_drain_whatif(N_S) restarts; U_S, the pinned request rows whose
 * leader is on N_S or whose `group` field names a restarted group; the placement what-if round with N_S
 * cordoned and U_S unpinned, diffed against the baseline placement rows.  Occupancy does not move, so the
 * answer is conservative, exactly as the per-key call is.  S TRIGGERS
 *   LWSE_DPW_LWS_FLOOR  when the set form lwse_resident_drain_budget over S has n_breached > 0;
 *   LWSE_DPW_STRANDED   when some row of U_S is not PLACED after;
 *   LWSE_DPW_BUMPED     when some row outside U_S is PLACED before and not after.
 * `constraints` (nonzero, known bits only) names the verdicts the plan keeps.  Keys are taken in the caller's
 * order and key k_i gets the first of:
 *   1. LWSE_DRAINW_BREACHES_ALONE  {k_i} triggers a verdict in constraints (wave LWSE_NONE);
 *   2. LWSE_DRAINW_PLANNED         wave w: the smallest index of an open wave such that W_w ∪ {k_i} triggers none
 *                                  of them; with no such wave and fewer than max_waves open, a new wave;
 *   3. LWSE_DRAINW_NO_WAVE         neither (wave LWSE_NONE).
 * Every wave is judged against the same baseline: the most recently submitted sweep and placement tick.
 *
 * The placement verdicts are NOT monotone in the set: draining more can unpin a pinned holder and free its
 * domain for a request another key stranded.  So a key that triggers alone is BREACHES_ALONE by definition even
 * when some wave would accept it, and the answer is the literal sequential first-fit, never a shortcut through
 * monotonicity.  Every returned wave's final key set was itself a probe (the probe of its last key), so every
 * wave is verified as a set: its row's placement counts are that probe's.
 *
 * Locality.  Per probe S = W ∪ {k} the call solves only the namespaces (a) holding a row of U_S, or (b) with a
 * baseline row that is not pinned and is PLACED in a domain d that S touches where S holds d as a domain key, or
 * the row's chosen node is in N_S, or dom_free[d] - sum of free[n] over the usable n in N_S ∩ d < size.  Every
 * other row keeps its baseline row.
 *
 * Readiness, isolation and errors: LWSE_ERR_NOT_READY when lwse_resident_drain_waves or
 * lwse_resident_drain_place_cost would answer it; LWSE_ERR_INVALID_ARG for a duplicate or out-of-range id, a
 * bad max_waves, NULL outputs, a nonzero reserved field, or a zero or unknown `constraints` bit;
 * LWSE_ERR_UNSUPPORTED with a peer exchange, at 2^24 resident requests or where the namespace form does not fit
 * the domains; LWSE_ERR_OOM when a sized scratch table refuses an entry.  A refused call writes no output.
 * Isolation as the other drain queries (the engine mutex, the what-if stream behind the snapshot event, scratch
 * that only grows, nothing of the tick touched).  n_ids = 0 is valid and opens no wave. */
#define LWSE_DPW_LWS_FLOOR (1u << 0)
#define LWSE_DPW_STRANDED (1u << 1)
#define LWSE_DPW_BUMPED (1u << 2)
#define LWSE_DPW_ALL (LWSE_DPW_LWS_FLOOR | LWSE_DPW_STRANDED | LWSE_DPW_BUMPED)

/* One key of the plan, in query order (48 B).  The floor alone columns equal row `id` of
 * lwse_resident_drain_budget_cost, the placement alone columns row `id` of lwse_resident_drain_place_cost. */
typedef struct lwse_drain_place_wave_key {
  uint32_t id;                /* the node row or domain id                                               */
  uint32_t wave;              /* its wave, or LWSE_NONE                                                  */
  uint32_t status;            /* LWSE_DRAINW_*                                                           */
  uint32_t alone;             /* the LWSE_DPW_* bits {id} triggers, whatever constraints holds           */
  uint32_t groups_restarted;  /* the key alone                                                           */
  uint32_t ready_restarted;
  uint32_t lws_touched;
  uint32_t lws_breached;
  uint32_t unpinned;          /* |U_k|                                                                   */
  uint32_t stranded;
  uint32_t bumped;
  uint32_t reserved;
} lwse_drain_place_wave_key;

/* One opened wave (96 B): the totals of lwse_resident_drain_budget and of the set-form drain placement over the
 * wave's ids.  The counts of verdicts in constraints are 0; the others report what the wave does to a verdict
 * the caller did not enforce. */
typedef struct lwse_drain_place_wave {
  uint32_t n_keys;
  uint32_t lws_touched;
  uint32_t lws_loses_available;
  uint32_t n_pods_evicted;
  uint32_t n_leaders_evicted;
  uint32_t n_groups_restarted;
  uint32_t n_ready_restarted;
  int32_t min_margin;         /* min over evaluated touched L of ready_after - floor; INT32_MAX for none */
  uint64_t n_pods_recreated;
  uint32_t lws_breached;
  uint32_t unpinned;          /* |U_S|                                                                   */
  uint32_t stranded;
  uint32_t bumped;
  uint32_t n_changed;         /* the lwse_place_whatif counters of the set-form composition              */
  uint32_t n_lost;
  uint32_t n_moved;
  uint32_t n_gained;
  uint32_t n_placed;
  uint32_t n_unschedulable;
  uint32_t n_conflict;
  uint32_t namespaces_solved; /* namespaces the wave's final probe solved                                */
  uint32_t reserved[2];
} lwse_drain_place_wave;

typedef struct lwse_drain_place_waves_query {
  /* in */
  const uint32_t* ids;              /* [n_ids] distinct node rows or domain ids (by scope), host memory    */
  uint32_t n_ids;
  uint32_t scope;                   /* LWSE_DRAIN_NODES or LWSE_DRAIN_DOMAINS                              */
  uint32_t max_waves;               /* 1 .. LWSE_DRAIN_WAVES_MAX                                           */
  uint32_t constraints;             /* LWSE_DPW_* (nonzero)                                                */
  uint32_t reserved;                /* 0                                                                   */
  uint32_t reserved1;               /* 0                                                                   */
  lwse_drain_place_wave_key* keys;  /* [n_ids] out                                                         */
  lwse_drain_place_wave* waves;     /* [max_waves] out: rows 0 .. n_waves                                  */
  /* out */
  uint32_t n_waves;
  uint32_t n_planned;
  uint32_t n_breaches_alone;
  uint32_t n_no_wave;
} lwse_drain_place_waves_query;
LWSE_API int lwse_resident_drain_place_waves(lwse_engine* e, lwse_drain_place_waves_query* q);

/* ---- rollout placement --------------------------------------------------------------------------
 * "Do the groups this rollout adds find an exclusive domain?" — for a list of LeaderWorkerSets, resident rows or
 * proposed edits, in one call.  The forecasts (lwse_resident_forecast, lwse_resident_rollout_whatif) assume every
 * group the leader StatefulSet holds becomes ready; an exclusive group that finds no free domain in its namespace
 * stays Pending instead (DESIGN.md §3.5, "Rollout placement").
 *
 * Definition.  Entry i names a resident LWS row L_i, a namespace id ns_i < the resident n_namespaces and, when
 * `recs` is given, a proposal P_i (an lwse_lws_rec with the contract of lwse_resident_rollout_whatif); without
 * `recs` P_i is the resident row L_i.  Each entry is answered on its own, as if its rollout were the only change;
 * several entries may name the same row.
 *   1. F_i is lwse_resident_rollout_whatif's forecast row for (L_i, P_i) — with P_i = L_i, lwse_resident_forecast's
 *      row of L_i — and peak = F_i.peak_sts_replicas.
 *   2. E_i holds, ascending, every group index g in [0, peak) with g >= group_count of L_i, or whose group row
 *      group_base + g lacks LWSE_GRP_POD_PRESENT: the groups encode_place_requests gives a request once their
 *      leader pods exist.  Row j of E_i is the request {priority, group_key} = the encoder's mix of
 *      (P_i.uid_hash, g), group = group_base + g, ns = ns_i, size = P_i.size, leader_node = LWSE_NONE.
 *   3. The answer is lwse_resident_place_whatif with no segments, extra = E_i (extra row j has row index and key
 *      rn_reqs + j) and the resident n_namespaces.  It solves ns_i alone (every other row keeps its baseline row):
 *      one namespace per entry, none when E_i is empty.
 *   4. An entry is not solved, and gets a flag, when L_i lacks LWSE_LWS_EXCLUSIVE_TOPOLOGY (NOT_EXCLUSIVE), when
 *      F_i has LWSE_LWSF_BAD_TABLE or LWSE_LWSF_NOT_FORECAST (NOT_FORECAST), or when P_i changes `size` or the
 *      exclusive bit of L_i (NOT_MODELLED: the rolled groups would need new domains).  An UNFINISHED forecast is
 *      solved with the peak of the cycles it replayed.  fc_flags and peak are F_i's for every entry.
 *
 * Readiness, isolation and errors: LWSE_ERR_NOT_READY wherever lwse_resident_forecast, lwse_resident_rollout_whatif
 * or lwse_resident_place_whatif would return it; LWSE_ERR_INVALID_ARG for a NULL query or array (with n > 0),
 * misaligned recs, a row >= n_lws or ns_i >= the resident n_namespaces; LWSE_ERR_UNSUPPORTED, writing nothing, on
 * an engine with a peer exchange, when rn_reqs + max |E_i| reaches 2^24 (row keys are 24-bit), where the namespace
 * form does not fit the domains, and when the proposals' slots reach the forecast's limit; LWSE_ERR_OOM rather
 * than a wrong row when sized scratch refuses an entry.  The call holds the engine mutex and runs on the what-if
 * stream behind one event on the engine's stream: the forecast snapshot and the placement baseline both come from
 * the most recently submitted tick, in flight or not.  It touches no tick graph, arena, change list, table, output
 * row, occupancy counter, node index or tick info; its scratch only grows.  n == 0 is a valid empty answer.
 * A refused call writes neither the rows, the extra rows nor the totals. */
typedef struct lwse_rollout_place { /* 64 B */
  uint32_t flags;            /* LWSE_RPL_*                                                              */
  uint32_t fc_flags;         /* F_i.flags                                                               */
  int32_t peak;              /* F_i.peak_sts_replicas                                                   */
  uint32_t surge;            /* |E_i| (0 for an entry that is not solved)                               */
  uint32_t placed;           /* rows of E_i PLACED after                                                */
  uint32_t stranded;         /* rows of E_i not PLACED after                                            */
  uint32_t own_lost;         /* resident rows whose `group` lies in L_i's range, PLACED before, not after */
  uint32_t bumped;           /* other resident rows PLACED before and not after                         */
  uint32_t n_changed;        /* the lwse_place_whatif counters of the composed query                    */
  uint32_t n_lost;
  uint32_t n_moved;
  uint32_t n_gained;
  uint32_t n_placed;
  uint32_t n_unschedulable;
  uint32_t n_conflict;
  uint32_t namespaces_solved; /* 0 or 1                                                                 */
} lwse_rollout_place;

#define LWSE_RPL_SOLVED (1u << 0)        /* answered: the counters hold the composed query's              */
#define LWSE_RPL_NOT_EXCLUSIVE (1u << 1) /* L_i lacks LWSE_LWS_EXCLUSIVE_TOPOLOGY                          */
#define LWSE_RPL_NOT_FORECAST (1u << 2)  /* F_i has LWSE_LWSF_BAD_TABLE or LWSE_LWSF_NOT_FORECAST          */
#define LWSE_RPL_NOT_MODELLED (1u << 3)  /* P_i changes size or the exclusive bit                          */
#define LWSE_RPL_STRANDS (1u << 4)       /* stranded > 0                                                   */
#define LWSE_RPL_BUMPS (1u << 5)         /* bumped > 0                                                     */

typedef struct lwse_rollout_place_query {
  const uint32_t* rows;      /* [n] resident LWS rows                                                   */
  const uint32_t* ns;        /* [n] namespace ids                                                       */
  const lwse_lws_rec* recs;  /* [n] proposals, 16-byte aligned, or NULL: the resident rows              */
  uint32_t n;
  uint32_t reserved;         /* 0                                                                       */
  lwse_rollout_place* out;   /* [n] out, host memory                                                    */
  lwse_place_req* extra;     /* [extra_capacity] out, host memory, or NULL: the rows of every E_i, entry
                                after entry in query order (the first extra_capacity of n_surge rows)   */
  uint64_t extra_capacity;
  /* out */
  uint32_t n_solved;         /* entries with LWSE_RPL_SOLVED                                            */
  uint32_t n_strands;        /* entries with LWSE_RPL_STRANDS                                           */
  uint64_t n_surge;          /* sum of surge                                                            */
  uint64_t n_stranded;       /* sum of stranded                                                         */
} lwse_rollout_place_query;
LWSE_API int lwse_resident_rollout_place(lwse_engine* e, lwse_rollout_place_query* q);

/* ---- rollout placement waves --------------------------------------------------------------------
 * "Which of these rollouts can I push together so that the groups they add all find an exclusive domain?"  The
 * first-fit plan of the drain waves over the entries of lwse_resident_rollout_place, with the rollouts of one wave
 * solved together (DESIGN.md §3.5, "Rollout placement waves").
 *
 * Definition.  rows, ns and recs are the entries of lwse_resident_rollout_place, with the same contract, except
 * that the rows must be distinct.  E_i is that call's extra rows of entry i.  For a set S of entries the set form is
 * lwse_resident_place_whatif with no segments, the resident n_namespaces and extra = E_{i1} || E_{i2} || ... over
 * S in query order, diffed against the baseline.  A resident row is S's own when its `group` lies in the group
 * range of an entry of S whose ns is the row's namespace.  S TRIGGERS
 *   LWSE_RPW_STRANDED  when some extra row is not PLACED after;
 *   LWSE_RPW_BUMPED    when some resident row PLACED before is not PLACED after (own_lost or bumped).
 * `constraints` (nonzero, known bits only) names the verdicts the plan keeps.  Only entries that
 * lwse_resident_rollout_place marks LWSE_RPL_SOLVED take part.  Keys are taken in query order and key k_i gets the
 * first of:
 *   3. LWSE_ROLLW_NOT_SOLVED       the entry is not SOLVED (wave LWSE_NONE);
 *   1. LWSE_ROLLW_TRIGGERS_ALONE   {k_i} triggers a verdict in constraints (wave LWSE_NONE);
 *   0. LWSE_ROLLW_PLANNED          wave w: the lowest open wave such that W_w ∪ {k_i} triggers none of them; with
 *                                  no such wave and fewer than max_waves open, a new wave;
 *   2. LWSE_ROLLW_NO_WAVE          neither (wave LWSE_NONE).
 * Every wave is judged against the same baseline, the most recently submitted tick: the plan assumes that a
 * wave's rollouts finish, and their surge groups go away, before the next wave starts.  The rollouts of one wave
 * are modelled at their peaks at the same time, so the plan is conservative as lwse_resident_rollout_place is.
 * The placement verdicts are not monotone in the set, so a key that triggers alone is TRIGGERS_ALONE even when
 * some wave would take it; the answer is the literal first-fit.  The plan decomposes exactly by namespace: keys of
 * different namespaces never wait for each other (DESIGN.md §3.5).
 *
 * Readiness, isolation and errors are lwse_resident_rollout_place's, and: LWSE_ERR_INVALID_ARG for a duplicate
 * row, max_waves of 0 or above LWSE_DRAIN_WAVES_MAX, a zero or unknown `constraints` bit, a nonzero reserved field,
 * a NULL keys (n > 0) or waves; LWSE_ERR_UNSUPPORTED also when rn_reqs + the sum of |E_i| over the SOLVED entries
 * reaches 2^24 (checked before the plan).  A refused call writes no output.  n = 0 is valid and opens no wave. */
#define LWSE_RPW_STRANDED (1u << 0)
#define LWSE_RPW_BUMPED (1u << 1)
#define LWSE_RPW_ALL (LWSE_RPW_STRANDED | LWSE_RPW_BUMPED)

#define LWSE_ROLLW_PLANNED 0u        /* = LWSE_DRAINW_PLANNED */
#define LWSE_ROLLW_TRIGGERS_ALONE 1u /* = LWSE_DRAINW_BREACHES_ALONE */
#define LWSE_ROLLW_NO_WAVE 2u        /* = LWSE_DRAINW_NO_WAVE */
#define LWSE_ROLLW_NOT_SOLVED 3u

/* One key of the plan, in query order (16 B). */
typedef struct lwse_rollout_wave_key {
  uint32_t wave;              /* its wave, or LWSE_NONE                                                  */
  uint32_t status;            /* LWSE_ROLLW_*                                                            */
  uint32_t alone;             /* the LWSE_RPW_* bits {k_i} triggers, whatever constraints holds          */
  uint32_t reserved;
} lwse_rollout_wave_key;

/* One opened wave (64 B): the totals of the set form over the wave's final key set.  The counts of verdicts in
 * constraints are 0; the others report what the wave does to a verdict the caller did not enforce. */
typedef struct lwse_rollout_wave {
  uint32_t n_keys;
  uint32_t surge;             /* extra rows: placed + stranded                                           */
  uint32_t placed;
  uint32_t stranded;
  uint32_t own_lost;          /* the wave's own resident rows PLACED before and not after                */
  uint32_t bumped;            /* other resident rows PLACED before and not after                         */
  uint32_t n_changed;         /* the lwse_place_whatif counters of the set form                          */
  uint32_t n_lost;
  uint32_t n_moved;
  uint32_t n_gained;
  uint32_t n_placed;
  uint32_t n_unschedulable;
  uint32_t n_conflict;
  uint32_t namespaces;        /* distinct namespaces among the wave's entries                            */
  uint32_t reserved[2];
} lwse_rollout_wave;

typedef struct lwse_rollout_place_waves_query {
  /* in */
  const uint32_t* rows;             /* [n] distinct resident LWS rows                                      */
  const uint32_t* ns;               /* [n] namespace ids                                                   */
  const lwse_lws_rec* recs;         /* [n] proposals, 16-byte aligned, or NULL: the resident rows          */
  uint32_t n;
  uint32_t max_waves;               /* 1 .. LWSE_DRAIN_WAVES_MAX                                           */
  uint32_t constraints;             /* LWSE_RPW_* (nonzero)                                                */
  uint32_t reserved;                /* 0                                                                   */
  lwse_rollout_wave_key* keys;      /* [n] out                                                             */
  lwse_rollout_wave* waves;         /* [max_waves] out: rows 0 .. n_waves                                  */
  lwse_rollout_place* alone_rows;   /* [n] out, or NULL: lwse_resident_rollout_place's rows for the query  */
  /* out */
  uint32_t n_waves;
  uint32_t n_planned;
  uint32_t n_triggers_alone;
  uint32_t n_no_wave;
  uint32_t n_not_solved;
  uint32_t reserved1;
} lwse_rollout_place_waves_query;
LWSE_API int lwse_resident_rollout_place_waves(lwse_engine* e, lwse_rollout_place_waves_query* q);

/* ---- scale headroom -----------------------------------------------------------------------------
 * "How many replicas can this object go to right now before a group it adds finds no exclusive domain?" — the
 * capacity question of an autoscaler (the HPA behind the LeaderWorkerSet scale subresource), for a list of exclusive
 * LeaderWorkerSets in one call (DESIGN.md §3.5, "Scale headroom").
 *
 * Definition.  Entry i names a resident LWS row L_i, a namespace id ns_i < the resident n_namespaces and, with
 * `ceilings`, a ceiling c_i (negative: none).  Entries are answered each on its own, as lwse_resident_rollout_place
 * answers them; rows may repeat.  r0 = L_i.replicas.
 *   1. P_i(R) is L_i with replicas := R and every other field unchanged (a scale-only edit).
 *   2. E_i(R) holds, ascending, every group index g in [0, R) with g >= group_count, or whose group row lacks
 *      LWSE_GRP_POD_PRESENT; row j is built as lwse_resident_rollout_place builds its row j (the encoder's mix of
 *      (uid_hash, g), row index and key rn_reqs + j).
 *   3. R is clean when lwse_resident_place_whatif with no segments and extra = E_i(R), diffed against the baseline,
 *      triggers none of `constraints`: LWSE_RPW_STRANDED (always required: some extra row is not PLACED after) and,
 *      opt-in, LWSE_RPW_BUMPED (some resident row PLACED before is not PLACED after, own_lost or bumped).
 *   4. An entry is answered (LWSE_SHR_SOLVED) only when L_i is settled: exclusive (else NOT_EXCLUSIVE); its resident
 *      forecast row without BAD_TABLE / NOT_FORECAST (else NOT_FORECAST); and (else NOT_SETTLED) LWSE_LWS_STS_EXISTS
 *      without LWSE_LWS_UPDATED, sts_replicas == replicas, sts_partition == 0, partition == 0, a forecast row
 *      without ROLLING / UNFINISHED / HELD and with peak_sts_replicas == final_replicas == replicas.  On a settled
 *      row a scale-only edit to R >= r0 is Case 3 of rollingUpdateParameters: the rollout what-if's forecast of
 *      P_i(R) has peak R, so E_i(R) is lwse_resident_rollout_place's E for the proposal P_i(R).  (With a held
 *      partition the surge of calculateLWSUnreadyReplicas can lift the StatefulSet above R; hence the partition
 *      clauses.)
 *   5. R_pig is the smallest R with |E_i(R)| = n_domains + 1: each placed extra row holds a distinct (ns_i, domain)
 *      pair, so R_pig always strands.  C_i = min(c_i, R_pig - 1).  max_replicas is the largest R in [r0, C_i]
 *      that is clean (r0 when c_i <= r0 and r0 is clean), or -1 with LWSE_SHR_BLOCKED when r0 itself triggers.
 *   6. The clean R form an interval [r0, H] (DESIGN.md §3.5), so the device bisects (r0, C_i]: exact, in
 *      ceil(log2(C_i + 1 - r0)) rounds, plus one for the entries whose bisection ends below R_pig without probing it.
 * The row carries lwse_resident_rollout_place's counters at `probe`: H + 1, the first R that triggers (r0 when
 * BLOCKED); with LWSE_SHR_AT_CEILING (max_replicas = c_i, or r0 for a ceiling <= r0) at H itself.  STRANDS / BUMPS
 * are the verdicts of that probe, whatever `constraints` holds.  An entry that is not solved has max_replicas and
 * probe -1 and zero counters.
 *
 * Readiness, isolation and errors are lwse_resident_rollout_place's (the mutex; the what-if stream behind one event on
 * the engine's stream; a tick in flight is neither waited on nor touched), and: LWSE_ERR_INVALID_ARG for a
 * `constraints` without LWSE_RPW_STRANDED or with an unknown bit, a nonzero reserved field, a NULL out (n > 0);
 * LWSE_ERR_UNSUPPORTED on an engine with a peer exchange, when rn_reqs + max |E| reaches 2^24 and where the namespace
 * form does not fit the domains.  A refused call writes nothing.  n = 0 is a valid empty answer. */
typedef struct lwse_scale_headroom { /* 64 B */
  uint32_t flags;            /* LWSE_SHR_*                                                              */
  int32_t replicas;          /* r0                                                                      */
  int32_t max_replicas;      /* H, or -1                                                                */
  int32_t probe;             /* the R whose counters follow, or -1                                      */
  uint32_t surge;            /* lwse_rollout_place's counters of P_i(probe): |E_i(probe)|               */
  uint32_t placed;
  uint32_t stranded;
  uint32_t own_lost;
  uint32_t bumped;
  uint32_t n_changed;
  uint32_t n_lost;
  uint32_t n_moved;
  uint32_t n_gained;
  uint32_t n_placed;
  uint32_t n_unschedulable;
  uint32_t n_conflict;
} lwse_scale_headroom;

#define LWSE_SHR_SOLVED (1u << 0)        /* answered                                                      */
#define LWSE_SHR_NOT_EXCLUSIVE (1u << 1) /* L_i lacks LWSE_LWS_EXCLUSIVE_TOPOLOGY                          */
#define LWSE_SHR_NOT_FORECAST (1u << 2)  /* its forecast row has BAD_TABLE or NOT_FORECAST                 */
#define LWSE_SHR_NOT_SETTLED (1u << 3)   /* a rollout, a scale or a partition is in progress or held       */
#define LWSE_SHR_BLOCKED (1u << 4)       /* r0 itself triggers: max_replicas = -1                          */
#define LWSE_SHR_AT_CEILING (1u << 5)    /* max_replicas is the ceiling (or r0 for a ceiling <= r0)        */
#define LWSE_SHR_STRANDS (1u << 6)       /* the probe strands an extra row                                 */
#define LWSE_SHR_BUMPS (1u << 7)         /* the probe takes a resident row's domain (own_lost or bumped)   */

typedef struct lwse_scale_headroom_query {
  const uint32_t* rows;         /* [n] resident LWS rows                                                */
  const uint32_t* ns;           /* [n] namespace ids                                                    */
  const int32_t* ceilings;      /* [n] c_i (negative: none), or NULL: none                              */
  uint32_t n;
  uint32_t constraints;         /* LWSE_RPW_STRANDED, optionally | LWSE_RPW_BUMPED                      */
  uint32_t reserved;            /* 0                                                                    */
  uint32_t reserved1;           /* 0                                                                    */
  lwse_scale_headroom* out;     /* [n] out, host memory                                                 */
  lwse_rollout_place* current;  /* [n] out, or NULL: lwse_resident_rollout_place's rows of the resident rows */
  /* out */
  uint32_t n_solved;            /* entries with LWSE_SHR_SOLVED                                         */
  uint32_t n_blocked;
  uint32_t n_at_ceiling;
  uint32_t rounds;              /* bisection rounds the call ran (the final probe included)             */
  uint64_t headroom;            /* sum of max_replicas - r0 over the SOLVED entries that are not BLOCKED */
} lwse_scale_headroom_query;
LWSE_API int lwse_resident_scale_headroom(lwse_engine* e, lwse_scale_headroom_query* q);

/* ------------------------------------------------------------------------- */
/* Peer exchange: the multi-GPU placement step without a collective library  */
/* ------------------------------------------------------------------------- */
#define LWSE_MAX_RANKS 16u
#define LWSE_IPC_HANDLE_BYTES 64u /* sizeof(cudaIpcMemHandle_t) */

/* One process per GPU of one node.  Every rank creates its exchange buffer (room for
 * `world` parts of [n_nodes occupancy counters | reqs_per_part request rows], twice) and
 * gets an IPC handle for it; the caller all-gathers the handles (any transport — they are
 * 64 opaque bytes) and hands all of them to lwse_exchange_connect, which maps the peers'
 * buffers over NVLink.  lwse_upload_nodes must have been called (the layout depends on
 * n_nodes); one exchange per engine.  reqs_per_part = 0: the parts carry occupancy only
 * (lwse_reconcile_shared_device). */
LWSE_API int lwse_exchange_create(lwse_engine* e, uint32_t reqs_per_part, uint32_t world, uint32_t rank,
                                  void* handle_out /* LWSE_IPC_HANDLE_BYTES */);
LWSE_API int lwse_exchange_connect(lwse_engine* e, const void* handles /* world x LWSE_IPC_HANDLE_BYTES */);
/* bytes of one part: align16(n_nodes * 4) + reqs_per_part * sizeof(lwse_place_req) */
LWSE_API uint64_t lwse_exchange_part_bytes(const lwse_engine* e);

/* A reconcile tick of one shard (see lwse_reconcile_device): `d_local_part` — this rank's
 * [occupancy | request rows (unused rows: leader_node = LWSE_NONE, size = 0)] in device
 * memory — is pushed into every peer's buffer with peer stores and a per-source flag is
 * raised there; the same kernel waits for all sources' flags of this step; then the placement
 * round runs over the gathered parts exactly as lwse_place_gathered_device does (d_place_out:
 * world * reqs_per_part rows; every rank computes the same answer and keeps its own rows).
 * All of it on the engine's side stream, concurrently with the sweep of `d` on `stream`
 * (d == NULL: placement step only).  Every rank must call this the same number of times. */
LWSE_API int lwse_reconcile_exchanged_device(lwse_engine* e, const lwse_lws_tables* d, const void* d_local_part,
                                             uint32_t n_namespaces, lwse_place_out* d_place_out, void* stream);
/* The tick of a shard whose placement requests are LOCAL to the rank and whose node occupancy is
 * shared — the north star's "single all-gather of the per-node occupancy vector": ranks own disjoint
 * namespaces (exclusivity is per namespace, so their rounds are independent), every rank's pods load
 * the same nodes.  `d_local_occupancy` (n_nodes counters, this rank's pods) is pushed into every
 * peer's buffer with peer stores + flags (lwse_exchange_create with reqs_per_part = 0 is enough);
 * the round then solves the n_reqs local requests (grouped by namespace) against the SUM of all
 * ranks' counters, concurrently with the sweep of `d` (NULL: placement branch only).
 * flags: LWSE_SWEEP_PLACE_SCAN, LWSE_EXCHANGE_LAGGED.  Every rank must call it the same number of times. */
#define LWSE_EXCHANGE_LAGGED (1u << 16) /* solve against the snapshot every rank pushed in the PREVIOUS
                                           call (own part included): no rank waits for the slowest
                                           rank's launch of this tick; results lag remote occupancy
                                           changes by one tick (the first call is in step)           */
LWSE_API int lwse_reconcile_shared_device(lwse_engine* e, const lwse_lws_tables* d, const lwse_place_req* d_reqs,
                                          uint32_t n_reqs, const uint32_t* d_local_occupancy, uint32_t n_namespaces,
                                          lwse_place_out* d_place_out, uint32_t flags, void* stream);
/* *error_out = 1 if a wait for the peers ever timed out (2 s; a rank is gone).  Synchronizes. */
LWSE_API int lwse_exchange_status(lwse_engine* e, uint32_t* error_out);

/* ------------------------------------------------------------------------- */
/* DisaggregatedSet sweep                                                    */
/* ------------------------------------------------------------------------- */
#define LWSE_DS_MAX_ROLES 10u /* api/disaggregatedset/v1: 2..10 roles             */
/* The limits of one DS: n_roles <= LWSE_DS_MAX_ROLES counts the removed roles too (roles of old
 * revisions that left the spec), so a DS with 10 spec roles that renamed one has 11 and is past it;
 * n_old_revs <= LWSE_DS_MAX_OLD_REVS; n_spec_roles <= n_roles; both ranges inside their tables.
 * A DS past any of them is reported LWSE_DOUT_BAD_TABLE (LWSE_DSF_BAD_TABLE by the forecast), not
 * reconciled: its role and revision-role rows are neither read nor written by the sweep, the DS
 * tick or the forecast (their role_out / revrole_out rows keep what the output tables held), and
 * no other DS's results change. */

/* One DisaggregatedSet (32 B). */
typedef struct lwse_ds_rec {
  uint64_t uid_hash;
  uint32_t role_base;  /* first row in the role table                            */
  uint32_t n_roles;    /* spec roles first, then removed roles (executor.go:140) */
  uint32_t n_spec_roles;
  uint32_t rev_base;   /* first row in the revision-role table                   */
  uint32_t n_old_revs; /* old revisions, each n_roles consecutive rows; the new
                          revision's n_roles rows follow them                    */
  uint32_t flags;      /* LWSE_DS_* */
} lwse_ds_rec;

#define LWSE_DS_HAS_NEW_REVISION (1u << 0) /* GetRevisionRolesList newRevision != nil */

/* One role of a DS (16 B). */
typedef struct lwse_ds_role_rec {
  int32_t target_replicas; /* getTargetReplicas (nil → 1)                        */
  int32_t max_surge;
  int32_t max_unavailable;
  uint32_t flags;          /* LWSE_ROLE_* */
} lwse_ds_role_rec;

#define LWSE_ROLE_SURGE_IS_PERCENT (1u << 0)
#define LWSE_ROLE_UNAVAIL_IS_PERCENT (1u << 1)
#define LWSE_ROLE_HAS_ROLLING_CONFIG (1u << 2) /* rollingUpdateConfiguration != nil */
#define LWSE_ROLE_IN_SPEC (1u << 3)
#define LWSE_ROLE_SURGE_INVALID (1u << 4)   /* intstr error (ignored → 0, executor.go:249) */
#define LWSE_ROLE_UNAVAIL_INVALID (1u << 5)

/* One (revision, role) LWS child of a DS (16 B).  Rows of one DS: for each old
 * revision (in List order) n_roles rows in role order, then n_roles rows for
 * the new (target) revision. */
typedef struct lwse_ds_revrole_rec {
  int32_t replicas;         /* getLWSReplicas: *spec.replicas, nil → 1            */
  int32_t initial_replicas; /* initial-replicas annotation, or -1 when absent/unparsable */
  int32_t ready_replicas;   /* status.readyReplicas                               */
  uint32_t flags;           /* LWSE_RR_* | creation rank << LWSE_RR_TS_SHIFT      */
} lwse_ds_revrole_rec;

#define LWSE_RR_EXISTS (1u << 0)       /* this revision has an LWS for this role   */
#define LWSE_RR_REPLICAS_NIL (1u << 1) /* spec.replicas == nil (cleanup counts it as 0,
                                          disaggregatedset_controller.go:222-225) */
#define LWSE_RR_TS_SHIFT 2             /* 30-bit order-preserving rank of
                                          metadata.creationTimestamp (executor.go:283-302) */

/* Per DS (16 B). */
typedef struct lwse_ds_out {
  uint32_t flags;        /* LWSE_DOUT_* */
  uint32_t drained_revs; /* bit r: old revision r has every role at 0 → delete its LWS */
  uint32_t ready_revs;   /* bit r: old revision r is ready on all spec roles (its
                            services are kept, service_manager.go:174-189)          */
  uint32_t reserved;
} lwse_ds_out;

#define LWSE_DOUT_ROLLING (1u << 0)   /* old revisions still hold replicas → rolling path */
#define LWSE_DOUT_INIT (1u << 1)      /* …but no new revision yet → initRollingUpdate     */
#define LWSE_DOUT_STABLE (1u << 2)    /* isRevisionStable(newRevision)                    */
#define LWSE_DOUT_STEP (1u << 3)      /* ComputeNextStep returned a step                  */
#define LWSE_DOUT_COMPLETE (1u << 4)  /* ComputeNextStep returned nil                     */
#define LWSE_DOUT_NEW_READY (1u << 5) /* target revision ready on all roles → ensure services */
#define LWSE_DOUT_BAD_TABLE (1u << 6)
#define LWSE_DS_MAX_OLD_REVS 32u

/* Per role (8 B): the planner step. */
typedef struct lwse_ds_role_out {
  int32_t next_old; /* UpdateStep.Past[i] */
  int32_t next_new; /* UpdateStep.New[i]  */
} lwse_ds_role_out;

/* Per (revision, role): spec.replicas after this reconcile — scaleUpNew /
 * scaleDownOld / reconcileSimple — or -1 where no LWS exists and none is
 * created (4 B). */
typedef int32_t lwse_ds_revrole_out;

typedef struct lwse_ds_tables {
  const lwse_ds_rec* ds;
  uint32_t n_ds;
  const lwse_ds_role_rec* roles;
  uint32_t n_roles;
  const lwse_ds_revrole_rec* revroles;
  uint32_t n_revroles;
  lwse_ds_out* ds_out;              /* n_ds       */
  lwse_ds_role_out* role_out;       /* n_roles    */
  lwse_ds_revrole_out* revrole_out; /* n_revroles */
} lwse_ds_tables;

LWSE_API int lwse_sweep_ds_host(lwse_engine* e, const lwse_ds_tables* host_tables);
LWSE_API int lwse_sweep_ds_device(lwse_engine* e, const lwse_ds_tables* dev_tables, void* stream);

/* ---- resident DS tables and the DS tick ---------------------------------------------------
 * The DisaggregatedSet reconciler is a controller of its own (disaggregatedset_controller.go:55-126,
 * its watches :273): DS objects and their child LeaderWorkerSets in, no pods.  Its tables stay
 * resident like the LeaderWorkerSet tables, with their own tick: watch events in as row patches of
 * the three tables below, the DS rows whose decisions changed out.  Replaces, per reconcile pass,
 * the List of child LWS and the planner / executor arithmetic of every DS
 * (disaggregatedset_controller.go:95-112,137-186,203-236; executor.go:85-124,199-398; planner.go:61-352).
 *
 * Both calls run on a DS stream of their own and never wait for, drain or drop the LeaderWorkerSet
 * ticks in flight (the exception to the rule that every other lwse_resident_* call drains first);
 * they touch neither the tick graphs nor the patch arena.  A load may allocate device and pinned
 * memory (which waits for the device as cudaMalloc does, without dropping any tick's results). */
/* (tables LWSE_TABLE_DS, LWSE_TABLE_DS_ROLES, LWSE_TABLE_DS_REVROLES: see lwse_table) */

/* The outputs of a DS tick: views of engine-owned pinned memory, valid until the next
 * lwse_ds_resident_* call.  ds_out / role_out / revrole_out are the FULL output tables, kept
 * current: the rows of a listed DS are rewritten by the tick, every other DS's rows still hold its
 * (unchanged) results.  A caller reads a changed DS's role and revision-role results in place, at
 * that DS's role_base and rev_base. */
typedef struct lwse_ds_changes {
  const uint32_t* ds_rows;               /* [n_changed] DS rows whose decisions changed; order unspecified */
  uint32_t n_changed;
  uint32_t reserved;
  const lwse_ds_out* ds_out;             /* [n_ds]       */
  const lwse_ds_role_out* role_out;      /* [n_roles]    */
  const lwse_ds_revrole_out* revrole_out;/* [n_revroles] */
} lwse_ds_changes;

/* Copy the three input tables of `host` to the device; they stay resident, and earlier DS results
 * are forgotten (the next tick lists every DS).  Output pointers in `host` are ignored.  Table sizes
 * are fixed from here on: the caller reserves spare rows (a zeroed DS row is a vacant DS). */
LWSE_API int lwse_ds_resident_load(lwse_engine* e, const lwse_ds_tables* host);
/* One DS reconcile pass: apply the patch segments (tables LWSE_TABLE_DS*; LWSE_PATCH_RANGE allowed;
 * rows / values anywhere in host memory, at most LWSE_TICK_MAX_SEGS segments), sweep every DS over
 * the resident tables, and report the DS whose lwse_ds_out row, role_out rows or revrole_out rows
 * differ from the previous tick, plus every DS whose own lwse_ds_rec row was patched in this tick
 * (a DS moved to other rows could otherwise compare equal to what those rows held).  Returns once
 * the results are in pinned memory (it spins on a sequence word; no stream synchronize).
 * LWSE_ERR_NOT_READY before lwse_ds_resident_load; LWSE_ERR_INVALID_ARG for NULL pointers, an
 * unknown table, or a row at or beyond its table's size.  A failed call changes no table and no
 * output. */
LWSE_API int lwse_ds_resident_tick(lwse_engine* e, const lwse_patch_seg* segs, uint32_t n_segs, lwse_ds_changes* out);

/* ---- links from revision-role rows to resident child LeaderWorkerSets ----------------------
 * A DS's children are ordinary LeaderWorkerSets named <ds>-<revision>-<role> (GenerateName,
 * pkg/utils/disaggregatedset/utils.go:92-94).  When a child is also resident in this engine's LWS
 * tables, the LWS tick has already computed the status.readyReplicas the DS tick needs
 * (updateConditions, leaderworkerset_controller.go:478-480).  A link lets the DS tick read that value
 * on the device instead of waiting for the status write, the watch event and a revision-role patch.
 *
 * LWSE_TABLE_DS_LINKS has one row per revision-role row, patched only through lwse_ds_resident_tick
 * (scattered or as ranges).  lwse_ds_resident_load sets every lws_row to LWSE_NONE (the first tick
 * after a load can send the whole table as one range).  Only status.readyReplicas is linked:
 * replicas and initial replicas are spec fields the DS controller writes itself.
 *
 * The rule.  Revision-role row r with link (L, U) uses lws_out[L].ready_replicas of the resident LWS
 * results when ALL of these hold, and its own ready_replicas otherwise:
 *   - row r has LWSE_RR_EXISTS;
 *   - LWS tables are resident (lwse_resident_load) and an LWS sweep was enqueued after the load and
 *     after every patch of LWSE_TABLE_LWS rows that came without a sweep (lwse_resident_patch, or a
 *     tick with LWSE_TICK_NO_SWEEP): until then the results do not belong to the resident LWS rows
 *     (after a load they are all-ones rows);
 *   - L < n_lws of the resident LWS table;
 *   - the resident lwse_lws_rec[L].uid_hash == U (a row the LWS encoder has since given to another
 *     object is harmless);
 *   - lws_out[L].flags has none of LWSE_LOUT_IRREGULAR, _BAD_TABLE, _RUP_ERROR, _STATUS_ERROR: in each
 *     case the reference never reaches Status().Update (Reconcile returns at :159-163, or
 *     updateConditions fails), so the value the API server holds is the row's own one.
 * Both objects must be on one engine: a child resident on another rank stays unlinked.
 *
 * Which LWS results.  A DS tick that has received a link patch since its load reads the results of
 * everything enqueued on the engine's stream when it starts: the most recently submitted LWS tick (or
 * lwse_resident_sweep), in flight or not.  It orders itself behind that work with one event and still
 * never waits for, drains or drops an LWS tick, nor touches the tick graphs or the patch arena.  A DS
 * tick that never received a link patch since its load waits on nothing. */
typedef struct lwse_ds_link { /* 16 B */
  uint64_t lws_uid_hash;      /* uid_hash of the child LWS (as in lwse_lws_rec)                      */
  uint32_t lws_row;           /* its row in the resident LWS table, or LWSE_NONE: not linked        */
  uint32_t reserved;           /* 0 (a patch with another value is rejected: LWSE_ERR_INVALID_ARG)  */
} lwse_ds_link;

/* How the last successful DS tick read ready counts (read-only; nothing waits). */
typedef struct lwse_ds_tick_info { /* 24 B */
  uint32_t linked;            /* 1: it ran the linked sweep (a link patch since the DS load)         */
  uint32_t rows_from_lws;     /* existing revision-role rows that took the LWS tick's ready count    */
  uint32_t rows_fallback;     /* linked rows (lws_row != LWSE_NONE) that used their own ready count   */
                              /* (both counts cover the revision-role rows the sweep reads: the
                                 (n_old_revs + 1) * n_roles rows of each DS whose row is not
                                 LWSE_DOUT_BAD_TABLE; link rows outside them are not counted) */
  uint32_t reserved;
  uint64_t lws_ticks;         /* LWS ticks submitted (lwse_resident_tick*, _sweep) when it read the
                                 LWS rows; 0 for an unlinked tick                                   */
} lwse_ds_tick_info;
LWSE_API int lwse_ds_resident_tick_info(lwse_engine* e, lwse_ds_tick_info* info);

/* ---- rollout forecast ---------------------------------------------------------------------
 * The rest of every DS rollout, replayed on the device from the current rows: the reconcile cycles
 * the DS controller would run if every child became ready before each cycle (simulateAllReady,
 * executor_test.go:190-201).  One cycle of one DS, on a private copy of its rows:
 *   1. every existing revision-role row gets ready_replicas = replicas;
 *   2. the DS is swept with the arithmetic of lwse_sweep_ds_* (the same device code);
 *   3. old revisions in drained_revs are deleted: their rows stop existing;
 *   4. on LWSE_DOUT_INIT every existing old row gets initial_replicas = replicas (SetInitialReplicas,
 *      executor.go:100-112) and the DS gets LWSE_DS_HAS_NEW_REVISION;
 *   5. every existing row takes its revrole_out value as replicas (a nil spec.replicas takes a value);
 *      a new-revision row that does not exist and has revrole_out >= 0 is created with that value
 *      (initRollingUpdate at 0, or reconcileSimple creating a missing role).
 * The replay stops at the first cycle that changes nothing (no replica value, no created or deleted
 * row, no INIT), or after the cycle cap min(2*M + 12, LWSE_DS_FORECAST_MAX_CYCLES), M being the largest
 * of any role's target_replicas and any role's sum over the DS's existing rows of max(replicas,
 * initial_replicas) (ComputeAllSteps' 2*max + 10, planner.go:355-385, plus the INIT and cleanup
 * cycles).  Per role, old = sum of replicas over existing old-revision rows, new = the new revision's
 * replicas (0 when absent); sums are 64-bit and stored clamped to int32.  A DS that is not on the
 * rolling path (LWSE_DOUT_ROLLING of a sweep of its current rows) runs no cycle.  DS whose row ranges
 * overlap another DS's give unspecified results, as for the sweep. */
#define LWSE_DS_FORECAST_MAX_CYCLES 65536u

typedef struct lwse_ds_forecast { /* per DS, 16 B */
  uint32_t flags;      /* LWSE_DSF_* */
  uint32_t cycles;     /* cycles that changed something */
  uint32_t step_base;  /* first trajectory row of this DS: rows of the DS before it, in DS order
                          (saturates at 0xFFFFFFFF)                                           */
  uint32_t n_steps;    /* cycles that changed some role's old or new count: n_steps * n_roles rows */
} lwse_ds_forecast;

#define LWSE_DSF_ROLLING (1u << 0)    /* the current rows are on the rolling path                  */
#define LWSE_DSF_WAITING (1u << 1)    /* …with a new revision that is not stable: the first cycle
                                         assumes it becomes ready                                    */
#define LWSE_DSF_DONE (1u << 2)       /* rolling, and stopped with no old replicas left and every
                                         spec role's new count at its target                         */
#define LWSE_DSF_UNFINISHED (1u << 3) /* rolling, and stopped with work left or at the cycle cap    */
#define LWSE_DSF_TRUNCATED (1u << 4)  /* its trajectory did not fit in step_capacity: none of its
                                         rows were written (the summaries are exact)                 */
#define LWSE_DSF_BAD_TABLE (1u << 6)  /* as LWSE_DOUT_BAD_TABLE; nothing else is set               */

typedef struct lwse_ds_forecast_role { /* per role row, 16 B (zero for rows of no valid DS) */
  int32_t peak_replicas;   /* max of old + new now and of old_k + new_{k+1} over cycles k (scaleUpNew
                              runs before scaleDownOld, executor.go:163-166)                   */
  int32_t floor_available; /* min of old + new now and of old_{k+1} + new_k over cycles k (drained pods
                              are gone, new ones are not ready yet)                            */
  int32_t final_old;       /* old and new after the last cycle (now, for a DS that runs none)  */
  int32_t final_new;
} lwse_ds_forecast_role;

/* Trajectory rows are lwse_ds_role_out rows {next_old, next_new} = {old, new} after a cycle that
 * changed some role's count, one per role; a DS's n_steps * n_roles rows are contiguous at step_base,
 * step-major.  A DS whose rows do not all fit below step_capacity gets LWSE_DSF_TRUNCATED and writes
 * none; no row at or beyond step_capacity is written, and no DS writes outside its own n_steps * n_roles
 * rows (also where overlapping row ranges make the results unspecified). */
typedef struct lwse_ds_forecast_out {
  lwse_ds_forecast* ds;              /* [n_ds]                                                */
  lwse_ds_forecast_role* roles;      /* [n_roles]                                             */
  lwse_ds_role_out* steps;           /* [step_capacity], or NULL: summaries only              */
  uint32_t step_capacity;
  uint32_t n_steps_written;          /* out: trajectory rows written                          */
  uint64_t n_steps_needed;           /* out: rows every DS's trajectory needs                 */
} lwse_ds_forecast_out;

/* Stateless: host tables in (output pointers of `host` ignored), host outputs out.  LWSE_ERR_INVALID_ARG
 * for NULL tables or outputs. */
LWSE_API int lwse_ds_forecast_host(lwse_engine* e, const lwse_ds_tables* host, lwse_ds_forecast_out* out);
/* Over the resident DS tables as the last lwse_ds_resident_tick (or the load) left them.  Runs on the
 * DS stream under the engine mutex, with scratch of its own: it changes no resident table, no DS tick
 * output, change list or counter, and never drains or drops LeaderWorkerSet ticks.  Links are ignored
 * (the forecast assumes readiness).  The scratch is sized by the tables and by the trajectory rows
 * written (never by step_capacity) and only grows: a call that needs more of it than any call before
 * allocates device memory, which waits for the device as cudaMalloc / cudaFree do (as
 * lwse_ds_resident_load); every other call waits only on the DS stream.  LWSE_ERR_NOT_READY before
 * lwse_ds_resident_load; LWSE_ERR_INVALID_ARG for NULL outputs. */
LWSE_API int lwse_ds_resident_forecast(lwse_engine* e, lwse_ds_forecast_out* out);

/* ---- DS rollout what-if -------------------------------------------------------------------
 * What a proposed edit of a DisaggregatedSet would make the DS controller do, before the edit reaches the
 * API server: a new image (a template edit, so a new target revision), a scale, or new maxSurge /
 * maxUnavailable.  A query is a list of proposals, each answered on its own as if it were the only edit;
 * several proposals may name the same DS (to compare settings).  For proposal i on resident DS row D
 * (n roles, V old revisions, header flags h) the proposed rows P_i are:
 *   - BAD_TABLE: D's resident row fails the sweep's limits or range test.  now[i] = {LWSE_DOUT_BAD_TABLE,
 *     0, 0, 0}, fc.ds[i].flags = LWSE_DSF_BAD_TABLE, its role rows in now_roles and fc.roles are 0 and
 *     nothing is gathered.  (A vacant, zeroed row is answered as the sweep answers it.)
 *   - Roles: D's n resident role rows, or with LWSE_DSP_ROLES the n rows at q->roles[i*10 .. i*10+n),
 *     in the resident order (spec roles, then removed roles); n_spec_roles stays the resident one.  A
 *     scale (target_replicas) or new rollout settings: ComputeRevision hashes only role names and templates
 *     (utils.go:173-199), so neither changes the revision.
 *   - Revision-role rows without LWSE_DSP_NEW_REVISION: D's (V+1)*n rows as they are.
 *   - With LWSE_DSP_NEW_REVISION, when h has LWSE_DS_HAS_NEW_REVISION, the target revision retires:
 *     V' = V + 1; old revisions 0..V-1 as resident; old revision V is D's current new-revision rows,
 *     unchanged; the new revision's n rows are absent {0, -1, 0, 0}; LWSE_DS_HAS_NEW_REVISION is cleared.
 *     V' > LWSE_DS_MAX_OLD_REVS makes the proposal BAD_TABLE, as the sweep reports the re-encoded DS.
 *   - With LWSE_DSP_NEW_REVISION, without LWSE_DS_HAS_NEW_REVISION: the target revision has no children to
 *     retire; V' = V and the rows are unchanged.
 *   - Links: a proposed row copied from resident row r carries r's link row; rows the edit creates carry
 *     none.  `now` follows the DS tick's link state: the rows are linked only after a link patch since the
 *     DS load, and LWS results count only while the LWS tables are loaded and swept.
 * P_i is exactly what the encoder writes for the edited object (same children, new target revision) when
 * the retired revision's children come last in List order; any other List order only permutes old
 * revisions.
 *   - now[i], now_roles[i*10 + j]: the ds_out / role_out rows of the linked DS sweep of P_i with the DS
 *     tick's device code and link rule: what the DS controller does first.  The bits of drained_revs /
 *     ready_revs number P_i's old revisions (the retired revision is bit V).
 *   - fc: lwse_ds_resident_forecast's rules over P_i (links ignored, as there), into fc.ds[i] and
 *     fc.roles[i*10 + j].  Proposal i's trajectory rows are contiguous at step_base, the offsets running
 *     over the proposals in query order, with the TRUNCATED / step_capacity / n_steps_written /
 *     n_steps_needed contract of lwse_ds_forecast_out.
 * Role rows j >= n of a proposal read 0 in now_roles and fc.roles.
 * Readiness and errors: LWSE_ERR_NOT_READY before lwse_ds_resident_load.  LWSE_ERR_INVALID_ARG for a NULL q;
 * n > 0 with NULL proposals, now, fc.ds or fc.roles; a LWSE_DSP_ROLES proposal with NULL or misaligned roles;
 * ds >= n_ds; unknown flag bits; reserved != 0.  LWSE_ERR_UNSUPPORTED when n > LWSE_DS_WHATIF_MAX_PROPOSALS
 * (checked before any array is read: the gathered rows then always index with uint32).  A failed call
 * writes nothing; n == 0 is a valid empty answer.
 * Isolation as lwse_resident_ds_drain: the what-if stream under the engine mutex, behind an event on the DS
 * stream and one on the engine's stream (it sees the last DS tick and the most recently submitted LWS tick,
 * in flight or not), with scratch of its own that only grows.  It touches no tick, graph, arena, change
 * list, resident LWS or DS table, link table, DS tick output, mirror or marks, tick info or counter, and
 * never waits for, drains or drops an LWS tick.
 * Out of scope: edits that add, remove or rename a role (they change allRoleNames and the row layout;
 * re-encode the object and call lwse_ds_forecast_host), edits that move a role between the spec and the removed
 * roles (n_spec_roles stays the resident one), and DS whose children live on another rank (each
 * rank answers its own DS). */
typedef struct lwse_ds_proposal { /* 8 B */
  uint32_t ds;                    /* resident DS row */
  uint32_t flags;                 /* LWSE_DSP_* */
} lwse_ds_proposal;
#define LWSE_DSP_NEW_REVISION (1u << 0) /* the edit changes ComputeRevision(spec.roles): a template edit */
#define LWSE_DSP_ROLES (1u << 1)        /* proposal i's role rows are q->roles[i*LWSE_DS_MAX_ROLES ..]  */
/* floor((2^32 - 1) / ((LWSE_DS_MAX_OLD_REVS + 1) * LWSE_DS_MAX_ROLES)) */
#define LWSE_DS_WHATIF_MAX_PROPOSALS 13015052u

typedef struct lwse_ds_rollout_whatif {
  const lwse_ds_proposal* proposals; /* [n] */
  const lwse_ds_role_rec* roles;     /* [n * LWSE_DS_MAX_ROLES], 16-byte aligned; read only for LWSE_DSP_ROLES
                                        proposals (may be NULL when none has it) */
  uint32_t n;
  uint32_t reserved;                 /* 0 */
  lwse_ds_out* now;                  /* [n] out */
  lwse_ds_role_out* now_roles;       /* [n * LWSE_DS_MAX_ROLES] out, or NULL */
  lwse_ds_forecast_out fc;           /* fc.ds [n], fc.roles [n * LWSE_DS_MAX_ROLES], fc.steps [step_capacity] or
                                        NULL */
} lwse_ds_rollout_whatif;
LWSE_API int lwse_resident_ds_rollout_whatif(lwse_engine* e, lwse_ds_rollout_whatif* q);

/* ---- DS drain ------------------------------------------------------------------------------
 * "Does this drain take an inference service down, or stall its rollout?"  A DisaggregatedSet serves
 * while every spec role of a revision has a ready replica (service_manager.go:57-89, :174-189: the sweep's
 * LWSE_DOUT_NEW_READY and ready_revs), and its rollout advances only while the target revision is stable,
 * replicas == readyReplicas on every spec role (isRevisionStable, executor.go:270-281: LWSE_DOUT_STABLE).
 * A drain can break either while every child LeaderWorkerSet stays above its own drain-budget floor.  The
 * reference has no drain logic: the definition below is this build's own (DESIGN.md §3.5, "DS drain").
 *
 * Definition.  Drain sets and lost(L, D) are those of lwse_resident_drain_budget: lost(L, D) is the number
 * of groups of LWS row L restarted by D whose baseline group row has LWSE_GOUT_COND_READY, against the
 * results of the most recently submitted LWS sweep.  For a revision-role row r of a DS that is not
 * LWSE_DOUT_BAD_TABLE, among the (n_old_revs + 1) * n_roles rows the sweep reads:
 *   ready_before(r)  the value the linked DS sweep reads (the link rule of lwse_ds_link): the child's baseline
 *                    lws_out[L].ready_replicas when r TAKES THE LWS VALUE, else r's own ready_replicas;
 *   ready_after(r)   ready_before(r) - lost(L, D) for a row that takes the LWS value (computed in 64 bits,
 *                    clamped to int32; several rows linked to one L all see the same lost), else ready_before.
 * The BEFORE and AFTER sweeps are linked DS sweeps of the resident DS tables (the DS tick's device code) with
 * ready_before and with ready_after.  "Before" is recomputed from the current LWS baseline, not read from the
 * last DS tick, so the two differ by the drain alone.  Per DS:
 *   LWSE_DSD_TOUCHED           some row that takes the LWS value has lost > 0;
 *   LWSE_DSD_SERVICE_LOST      NEW_READY before, not after;
 *   LWSE_DSD_OLD_SERVICE_LOST  ready_revs before & ~ready_revs after != 0;
 *   LWSE_DSD_STALLS            STABLE before, not after;
 *   LWSE_DSD_CHANGED           a ds_out row, or (not BAD_TABLE) a role_out or revrole_out row of the DS differs.
 *   rows_touched               rows that take the LWS value and have lost > 0 (removed roles included);
 *   rows_zeroed                of those, the rows with ready_before >= 1 and ready_after < 1.
 * Only the ready column moves between the two sweeps, so a DS that is not touched is not changed either.
 *
 * Readiness and errors: LWSE_ERR_NOT_READY unless the drain budget is ready (as lwse_resident_drain_budget)
 * and DS tables are resident (lwse_ds_resident_load).  With no link patch since the DS load every row falls
 * back: nothing is touched and rows_linked is 0.  LWSE_ERR_INVALID_ARG as for lwse_resident_drain_budget.
 * Isolation: the what-if stream under the engine mutex, behind an event on the engine's stream and one on
 * the DS stream, with scratch of its own that only grows; no tick, graph, arena, change list, resident LWS
 * or DS table, DS tick output or mirror, link table, occupancy counter, node index or tick info is touched.
 * Multi-rank engines: a DS and its children live on one rank, so every count sums over the ranks.  DS whose row
 * ranges overlap give results as unspecified as the sweep's; every write of both calls stays in their scratch
 * (a row read by k DS counts k times, and the per-key form sizes its scratch from that count). */
#define LWSE_DSD_TOUCHED (1u << 0)
#define LWSE_DSD_SERVICE_LOST (1u << 1)
#define LWSE_DSD_OLD_SERVICE_LOST (1u << 2)
#define LWSE_DSD_STALLS (1u << 3)
#define LWSE_DSD_CHANGED (1u << 4)

/* One touched DS of a drain (64 B). */
typedef struct lwse_ds_drain {
  uint32_t ds;                /* DS row                                                                  */
  uint32_t flags;             /* LWSE_DSD_*                                                              */
  uint32_t rows_touched;
  uint32_t rows_zeroed;
  uint32_t new_zeroed_roles;  /* bit i: spec role i's row of the new revision is zeroed (the roles that take
                                 its service down when SERVICE_LOST)                                     */
  uint32_t old_zeroed_roles;  /* bit i: spec role i is zeroed in an old revision whose ready_revs bit falls
                                 (the union over those revisions)                                        */
  uint32_t reserved[2];
  lwse_ds_out before;         /* its ds_out row in the before and the after sweep                        */
  lwse_ds_out after;
} lwse_ds_drain;

/* The set form: the touched DS of one drain set, and its totals. */
typedef struct lwse_ds_drain_query {
  /* in */
  const uint32_t* ids;        /* [n_ids] node rows or domain ids (by scope), host memory; duplicates allowed */
  uint32_t n_ids;
  uint32_t scope;             /* LWSE_DRAIN_NODES or LWSE_DRAIN_DOMAINS                                  */
  uint32_t capacity;          /* rows `rows` holds                                                       */
  uint32_t reserved;
  lwse_ds_drain* rows;        /* [capacity]: touched DS (beyond capacity not listed; order unspecified)  */
  lwse_ds_role_out* role_out; /* [n_roles] or NULL: the after sweep's full role_out (rows no DS's sweep
                                 writes read 0)                                                          */
  lwse_ds_revrole_out* revrole_out; /* [n_revroles] or NULL: the after sweep's full revrole_out (as role_out) */
  /* out */
  uint32_t n_touched;         /* every touched DS, listed or not                                         */
  uint32_t n_service_lost;
  uint32_t n_old_service_lost;
  uint32_t n_stalled;
  uint32_t n_changed;
  uint32_t rows_touched;      /* summed over the touched DS                                              */
  uint32_t rows_zeroed;
  uint32_t rows_linked;       /* rows that take the LWS value, touched or not                            */
} lwse_ds_drain_query;
LWSE_API int lwse_resident_ds_drain(lwse_engine* e, lwse_ds_drain_query* q);

/* The per-key form: one row per node (LWSE_DRAIN_NODES, n_nodes rows) or per domain (LWSE_DRAIN_DOMAINS,
 * n_domains rows), row k holding what lwse_resident_ds_drain gives for the node k or the nodes of domain k
 * (32 B; LWSE_DSD_CHANGED has no column: it needs the whole sweep).  Exact in one pass: lost(L, k) is the
 * drain budget's per-key count, and only the ready column differs between the two sweeps, so NEW_READY
 * falls iff a spec row of the new revision has ready_before >= 1 > ready_after, an old revision's ready bit
 * iff one of its spec rows does, and STABLE iff a spec row of the new revision changes its ready count (before
 * the drain ready == replicas there).  Each verdict is an OR over (row, key) facts gated by the DS's flags in
 * the before sweep.  The (LWS, key) and (DS, key) pairs are gathered in open-addressing tables in scratch,
 * each sized from a counting pass (one host synchronisation each); an insert a table refuses fails the call
 * with LWSE_ERR_OOM.  Readiness, isolation and errors as lwse_resident_ds_drain; `out` is host memory. */
typedef struct lwse_ds_drain_cost {
  uint32_t ds_touched;        /* n_touched of the set form for this key                                  */
  uint32_t ds_service_lost;
  uint32_t ds_old_service_lost;
  uint32_t ds_stalled;
  uint32_t rows_touched;
  uint32_t rows_zeroed;
  uint32_t reserved[2];
} lwse_ds_drain_cost;
LWSE_API int lwse_resident_ds_drain_cost(lwse_engine* e, uint32_t scope, lwse_ds_drain_cost* out);

/* ---- DS drain waves ------------------------------------------------------------------------
 * "Which of these nodes (domains) can I drain together and keep every inference service up?"  The first-fit plan
 * of lwse_resident_drain_waves with a wave rule that also reads the DS verdicts of lwse_resident_ds_drain
 * (DESIGN.md §3.5, "DS drain waves").  A child LeaderWorkerSet with replicas 1 and maxUnavailable 1 has floor 0:
 * the LWS rule lets a wave take its only replica, and the DS that reads it stops serving.
 *
 * Definition.  ids, scope, max_waves, drain sets, EVALUATED, floor, ready_before and lost(L, D) are those of
 * lwse_resident_drain_waves; TOUCHED, SERVICE_LOST, OLD_SERVICE_LOST and STALLS those of lwse_resident_ds_drain.
 * A drain set D TRIGGERS
 *   LWSE_DSW_LWS_FLOOR       when the set form lwse_resident_drain_budget over D has n_breached > 0;
 *   LWSE_DSW_DS_SERVICE      when lwse_resident_ds_drain over D has n_service_lost > 0;
 *   LWSE_DSW_DS_OLD_SERVICE  when it has n_old_service_lost > 0;
 *   LWSE_DSW_DS_STALL        when it has n_stalled > 0.
 * `constraints` (nonzero, known bits only) names the verdicts the plan keeps.  Keys are taken in the caller's
 * order and key k_i gets the first of:
 *   1. LWSE_DRAINW_BREACHES_ALONE  {k_i} triggers a verdict in constraints (wave LWSE_NONE);
 *   2. LWSE_DRAINW_PLANNED         wave w: the smallest index of an open wave such that W_w ∪ {k_i} triggers none
 *                                  of them; with no such wave and fewer than max_waves open, a new wave;
 *   3. LWSE_DRAINW_NO_WAVE         neither (wave LWSE_NONE).
 * Every wave is judged against the same baseline, as in lwse_resident_drain_waves.
 *
 * Exact through one cap per LWS row.  A revision-role row r that takes the LWS value of child L (the link rule of
 * lwse_ds_link) has ready_before(r) = lws_out[L].ready_replicas and ready_after(r) = ready_before - lost(L, D), so
 * every row linked to L moves together.  Each DS verdict is an OR over its rows, gated by the DS's flags in the
 * before sweep (see lwse_resident_ds_drain_cost), and is monotone in D.  A gated row therefore bounds lost(L, D):
 *   - a new-revision spec row of a DS with NEW_READY before (SERVICE), or a spec row of old revision v of a DS with
 *     bit v of ready_revs before (OLD_SERVICE): lost(L, D) <= ready_before - 1;
 *   - a new-revision spec row of a DS with STABLE before (STALL; only a DS mid-rollout is STABLE): lost(L, D) = 0.
 * Removed roles, rows that fall back and rows of BAD_TABLE DS bound nothing.  With slack(L) the minimum of
 * ready_before - floor (LWS_FLOOR in constraints and L EVALUATED), ready_before - 1 (L linked from a row whose
 * verdict is in constraints and gated) and 0 (STALL, likewise), +inf otherwise, adding k to W is admissible iff
 * every L to which k adds new > 0 ready member groups has lost(L, W) + new <= slack(L).  Unlike the LWS plan, the
 * groups of L count whether or not L is EVALUATED whenever some row the DS sweep reads takes L's value: the DS
 * verdicts read lost(L, ·) for such an L either way.  With no link patch since the DS load no row takes an LWS
 * value and the DS constraints bind nothing.
 *
 * Readiness, isolation and errors: as lwse_resident_ds_drain (LWSE_ERR_NOT_READY without a ready drain budget and
 * resident DS tables; the what-if stream behind the engine-stream and DS-stream events; scratch of its own that
 * only grows), plus the refusals of lwse_resident_drain_waves: LWSE_ERR_INVALID_ARG for a duplicate or
 * out-of-range id, a bad max_waves, NULL outputs, a nonzero reserved field or a zero or unknown `constraints`
 * bit; LWSE_ERR_UNSUPPORTED with a peer exchange; LWSE_ERR_OOM when a sized scratch table refuses an entry.  A
 * refused call writes no output.  n_ids = 0 is valid and opens no wave. */
#define LWSE_DSW_LWS_FLOOR (1u << 0)
#define LWSE_DSW_DS_SERVICE (1u << 1)
#define LWSE_DSW_DS_OLD_SERVICE (1u << 2)
#define LWSE_DSW_DS_STALL (1u << 3)
#define LWSE_DSW_ALL (LWSE_DSW_LWS_FLOOR | LWSE_DSW_DS_SERVICE | LWSE_DSW_DS_OLD_SERVICE | LWSE_DSW_DS_STALL)

/* One key of the plan, in query order (48 B).  The alone columns equal row `id` of
 * lwse_resident_drain_budget_cost and of lwse_resident_ds_drain_cost for the same scope. */
typedef struct lwse_ds_drain_wave_key {
  uint32_t id;                  /* the node row or domain id                                             */
  uint32_t wave;                /* its wave, or LWSE_NONE                                                */
  uint32_t status;              /* LWSE_DRAINW_*                                                         */
  uint32_t alone;               /* the LWSE_DSW_* bits {id} triggers, whatever constraints holds         */
  uint32_t groups_restarted;    /* the key alone                                                         */
  uint32_t ready_restarted;
  uint32_t lws_touched;
  uint32_t lws_breached;
  uint32_t ds_touched;
  uint32_t ds_service_lost;
  uint32_t ds_old_service_lost;
  uint32_t ds_stalled;
} lwse_ds_drain_wave_key;

/* One opened wave (80 B): the totals of lwse_resident_drain_budget and of lwse_resident_ds_drain over the wave's
 * ids.  The counts of verdicts in constraints are 0; the others report what the wave does to a verdict the caller
 * did not enforce. */
typedef struct lwse_ds_drain_wave {
  uint32_t n_keys;
  uint32_t lws_touched;
  uint32_t lws_breached;
  uint32_t lws_loses_available;
  uint32_t n_pods_evicted;
  uint32_t n_leaders_evicted;
  uint32_t n_groups_restarted;
  uint32_t n_ready_restarted;
  int32_t min_margin;           /* min over evaluated touched L of ready_after - floor; INT32_MAX for none */
  uint32_t ds_touched;
  uint32_t ds_service_lost;
  uint32_t ds_old_service_lost;
  uint32_t ds_stalled;
  uint32_t rows_touched;
  uint32_t rows_zeroed;
  uint32_t reserved;
  uint64_t n_pods_recreated;
  uint64_t reserved2;
} lwse_ds_drain_wave;

typedef struct lwse_ds_drain_waves_query {
  /* in */
  const uint32_t* ids;           /* [n_ids] distinct node rows or domain ids (by scope), host memory       */
  uint32_t n_ids;
  uint32_t scope;                /* LWSE_DRAIN_NODES or LWSE_DRAIN_DOMAINS                                 */
  uint32_t max_waves;            /* 1 .. LWSE_DRAIN_WAVES_MAX                                              */
  uint32_t constraints;          /* LWSE_DSW_* (nonzero)                                                   */
  uint32_t reserved;             /* 0                                                                      */
  uint32_t reserved1;            /* 0                                                                      */
  lwse_ds_drain_wave_key* keys;  /* [n_ids] out                                                            */
  lwse_ds_drain_wave* waves;     /* [max_waves] out: rows 0 .. n_waves                                     */
  /* out */
  uint32_t n_waves;
  uint32_t n_planned;
  uint32_t n_breaches_alone;
  uint32_t n_no_wave;
} lwse_ds_drain_waves_query;
LWSE_API int lwse_resident_ds_drain_waves(lwse_engine* e, lwse_ds_drain_waves_query* q);

/* ------------------------------------------------------------------------- */
/* Group / subgroup keys (SHA-1) and subgroup indices                        */
/* ------------------------------------------------------------------------- */
/* keys: n strings, string i = bytes[offsets[i] .. offsets[i+1]) (the caller
 * formats "<ns>/<podName>" or "<leaderName>/<subIdx>"); digests: n x 20 bytes. */
LWSE_API int lwse_group_keys_host(lwse_engine* e, const uint8_t* bytes, const uint32_t* offsets,
                                  uint32_t n, uint8_t* digests);
LWSE_API int lwse_group_keys_device(lwse_engine* e, const uint8_t* d_bytes,
                                    const uint32_t* d_offsets, uint32_t n, uint8_t* d_digests,
                                    void* stream);

/* Subgroup indices and subgroup keys of n pods in one pass (pod_webhook.go:249-255
 * getSubGroupIndex, :130/:151 the subgroup key): pod i has leader-pod name
 * bytes[offsets[i] .. offsets[i+1]), group size pod_count[i], subgroup size subgroup_size[i] and
 * worker index worker_index[i].  index_out[i] = getSubGroupIndex(...) with Go's truncating
 * division (worker 0 of a "leader is extra" group with subgroup size 1 gives -1, as the Go
 * expression does); digests[i] = SHA-1("<leaderName>/<index>") — the "/<index>" suffix is formed on
 * the device.  subgroup_size[i] == 0 (a division by zero in Go): index_out[i] = INT32_MIN and a
 * zero digest. */
LWSE_API int lwse_subgroup_keys_host(lwse_engine* e, const uint8_t* bytes, const uint32_t* offsets, uint32_t n,
                                     const int32_t* pod_count, const int32_t* subgroup_size,
                                     const int32_t* worker_index, int32_t* index_out, uint8_t* digests);
LWSE_API int lwse_subgroup_keys_device(lwse_engine* e, const uint8_t* d_bytes, const uint32_t* d_offsets, uint32_t n,
                                       const int32_t* d_pod_count, const int32_t* d_subgroup_size,
                                       const int32_t* d_worker_index, int32_t* d_index_out, uint8_t* d_digests,
                                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LWSE_H_ */
