// vr_tree.h -- the device tree behind the C-ABI's vr_tree handle and the CUDA error channel, shared by the tree's
// construction (vr_tree.cu) and the launch entry points (vr_api.cu).  No other file includes it.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <mutex>
#include <unordered_map>

#include "vr_frames.h"
#include "vr_types.h"
#include "vr_wire.h"

namespace vrb {

// Kernel launches so far (vr_launch_count): every entry point adds the launches it makes.
extern std::atomic<unsigned long long> g_launches;

// The device check of every entry point.  With a tree, the current device must be the tree's (cudaGetDevice only, so
// launches pay no more); without one, some device must exist.
int need_device(const vr_tree* t);

// A buffer a kernel dereferences: NULL, or memory the tree's device can address (not pageable host memory, not another
// device's allocation); `what` names it in the error.
int buffer_check(const vr_tree* t, const void* p, const char* what);

// The table entry -> slot map (VR_TREE_SLOT_MAP) of the operations on leaf slots: VR_EUNSUPPORTED without it; `what`
// names the operation in the error.
int need_slot_map(const vr_tree* t, const char* what);

// A failed CUDA call: VR_ENOMEM for an allocation, else VR_ECUDA, with the message "<what>: <CUDA's text><where>".
// The runtime's last error is cleared, so that a later launch check does not report this failure again.
inline int cuda_fail(cudaError_t e, const char* what, const char* where = "") {
    cudaGetLastError();
    return fail(e == cudaErrorMemoryAllocation ? VR_ENOMEM : VR_ECUDA, "%s: %s%s", what, cudaGetErrorString(e), where);
}

}  // namespace vrb

#define VR_STR_(x) #x
#define VR_STR(x) VR_STR_(x)
#define VR_CUDA(expr)                                                                                          \
    do {                                                                                                       \
        const cudaError_t e__ = (expr);                                                                        \
        if (e__ != cudaSuccess) return vrb::cuda_fail(e__, #expr, " (" __FILE__ ":" VR_STR(__LINE__) ")"); \
    } while (0)

// Per-stream launch resources of a tree.  Work-queue slots and the camera ring are recycled in
// stream order only: a launch that reuses a slot is ordered behind the launch that used it before, so
// no fence is needed, and launches on different streams never share a slot.
struct StreamRes {
    unsigned int* queues = nullptr;  // kQueueSlots slots of kQueueSlotBytes: {head, done}, per-SM block states and locks (vr_march.cuh)
    vrb::CamDev* cam_ring = nullptr; // kCamRing entries; batches take consecutive slots
    vrb::OptDev* opt_ring = nullptr; // kCamRing entries beside cam_ring (same slots), allocated by the first
                                     // batch with options per view
    unsigned int next_queue = 0, cam_pos = 0;
    unsigned long long data_gen = 0; // the tree's data_gen at this stream's last march launch
};

struct vr_tree {
    int device = 0;
    int num_sms = 0;
    vrb::TreeDev dev{};
    uint32_t* wide = nullptr;
    unsigned char* wrecs = nullptr;
    float* extra = nullptr;
    // upload scratch (slot-indexed node words, table entry -> slot), freed once the tables are built; with
    // VR_TREE_SLOT_MAP the table entry -> slot map stays (vr_tree_leaf_weights, vr_tree_leaf_grads, vr_tree_update_data)
    uint32_t* nodes = nullptr;
    uint32_t* wslot = nullptr;
    long long n_tables = 0;
    std::mutex res_mu;
    std::unordered_map<cudaStream_t, StreamRes> res;
    // bumped (under res_mu) by every vr_tree_update_data: a stream's first march launch after an update is made
    // without programmatic dependent launch, since the march reads the tree before griddepcontrol.wait (dispatch)
    unsigned long long data_gen = 0;
    // vr_render_frames_host: chunk ring, streams and events are created once and kept
    struct HostPath {
        static constexpr int kRing = 4;
        uint8_t* buf[kRing] = {};
        size_t buf_bytes = 0;
        cudaEvent_t rendered[kRing] = {}, copied[kRing] = {};
        cudaStream_t sr[2] = {nullptr, nullptr}, sc = nullptr;
        bool ready = false;
    } host;
    std::mutex host_mu;
    vr_tree_info info{};
    int data_dim = 0;
    // grid wireframe (vr_tree_wireframe): cells per level, counted on the first call
    std::mutex wire_mu;
    bool wire_ready = false;
    vrb::WireLevels wire_levels{};
};
