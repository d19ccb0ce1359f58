// The restart verdict of handleRestartPolicy (pod_controller.go:204-266) for one pod group (sm_90a):
// the group-level gate (policy and pending state, :209-226) and the per-pod predicate
// (workerPodBelongsToLeader :268-295, the revision check :233-239).  Shared by the group pass
// (lwse_lws_kernels.cu) and the drain cost (lwse_drain_kernels.cu), so that the cost evaluates
// the sweep's own predicate.
#pragma once

#include "lwse_device.cuh"

namespace lwse {

// What deciding one event pod needs from its group (pod_controller.go:233-257).
struct VisitCtx {
  uint32_t rev_lo, rev_hi;  // leader pod's revision hash
  uint32_t leader_uid, wsts_uid;
  uint32_t pod_base;
  uint32_t bits;  // kLeaderFound | kChainOk | kLeaderDeleting
};
constexpr uint32_t kLeaderFound = 1u, kChainOk = 2u, kLeaderDeleting = 4u;
constexpr uint32_t kAccLeaderCand = 0x80000000u;

// RecreateGroupOnPodRestart or RecreateGroupAfterStart: the policy visits event pods at all (:209).
__device__ __forceinline__ bool restart_policy_on(uint32_t lflags) {
  const uint32_t policy = (lflags & LWSE_LWS_RESTART_MASK) >> LWSE_LWS_RESTART_SHIFT;
  return policy == LWSE_RESTART_ON_POD_RESTART || policy == LWSE_RESTART_AFTER_START;
}

// :222 skip when pendingPodsInGroup ∧ (AfterStart ∨ the recreate-after-start annotation)
__device__ __forceinline__ bool restart_suppressed(bool pending, uint32_t lflags) {
  const uint32_t policy = (lflags & LWSE_LWS_RESTART_MASK) >> LWSE_LWS_RESTART_SHIFT;
  return pending && (policy == LWSE_RESTART_AFTER_START || (lflags & LWSE_LWS_RECREATE_AFTER_START_ANNOT));
}

// The group's part of the per-pod predicate, from its 64-byte row (ca..cd).
__device__ __forceinline__ void visit_ctx_of(VisitCtx& c, const uint4 ca, const uint4 cb, const uint4 cc, const uint4 cd) {
  const uint32_t gflags = cd.y;
  constexpr uint32_t kChain = LWSE_GRP_WSTS_FOUND | LWSE_GRP_WSTS_OWNER_IS_POD | LWSE_GRP_WSTS_OWNER_NAME_MATCH;
  c.rev_lo = ca.x;
  c.rev_hi = ca.y;
  c.leader_uid = cb.z;
  c.wsts_uid = cb.w;
  c.pod_base = cc.z;
  c.bits = 0;
  if ((gflags & (LWSE_GRP_POD_PRESENT | LWSE_GRP_POD_NAME_MATCH)) == (LWSE_GRP_POD_PRESENT | LWSE_GRP_POD_NAME_MATCH))
    c.bits |= kLeaderFound;  // :233
  if ((gflags & kChain) == kChain && cc.x == cb.z) c.bits |= kChainOk;  // sts owner uid == leader uid
  if (gflags & LWSE_GRP_POD_DELETING) c.bits |= kLeaderDeleting;
}

// handleRestartPolicy (:204-266) for ONE pod that has a restart / deletion event, policy checks
// already done: returns the verdict bits it contributes; *cand = it would recreate the group.
// *cand reads neither the pod's deleting bit nor the leader's: those only choose between
// DELETE_LEADER and LEADER_DELETING.
__device__ __forceinline__ uint32_t visit_pod(const VisitCtx& c, uint32_t state, const uint4 id, bool& cand) {
  uint32_t acc = 0;
  bool deleting;
  if (state & LWSE_POD_IS_LEADER) {
    cand = true;  // leader = pod (:251)
    deleting = state & LWSE_POD_DELETING;
    acc |= kAccLeaderCand;
  } else if (!(id.w & LWSE_PODID_NAME_OK)) {
    cand = false;
    return LWSE_GOUT_RESTART_ERROR;  // :230
  } else {
    const uint32_t kind = (state & LWSE_POD_OWNER_MASK) >> LWSE_POD_OWNER_SHIFT;
    // workerPodBelongsToLeader :268-295
    const bool belongs = (state & LWSE_POD_OWNER_NAME_MATCH) &&
                         ((kind == 1u && id.z == c.leader_uid) || (kind == 2u && id.z == c.wsts_uid && (c.bits & kChainOk)));
    cand = (c.bits & kLeaderFound) && id.x == c.rev_lo && id.y == c.rev_hi && belongs;  // :233, :239
    deleting = c.bits & kLeaderDeleting;
  }
  if (!cand) return 0;
  return acc | (deleting ? LWSE_GOUT_LEADER_DELETING : LWSE_GOUT_DELETE_LEADER);  // :255 / :259
}

}  // namespace lwse
