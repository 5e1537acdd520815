// vr_tree.h -- the device tree behind the C-ABI's vr_tree handle and the CUDA error channel, shared by the tree's
// construction (vr_tree.cu), its coarse sigma grid and the tile-coverage pass (vr_cull.cu) and the launch entry points
// (vr_api.cu).  No other file includes it.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <mutex>
#include <unordered_map>

#include "vr_frames.h"
#include "vr_types.h"
#include "vr_wire.h"

namespace vrb {

// Kernel launches so far (vr_launch_count): every entry point adds the launches it makes, except that a batch
// render's tile-coverage pass is counted with the march it prepares -- one count per march launch, as callers that
// budget launches per batch (one march per chunk) have always seen it.
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

// The coarse sigma grid of a tree from its tables (vr_cull.cu), ordered on `stream`.  with_org: first the origin of
// every table into t->tab_org (tree creation); without, the origins of the creation are reused (vr_tree_update_data,
// which changes sigma only).  Returns the number of kernels launched, or a negative value on a CUDA error.
int build_sigma_grid(vr_tree* t, cudaStream_t stream, bool with_org);

// The tile-coverage pass of a batch launch (vr_cull.cu): writes the tile mask of P's n_views views into the stream's
// mask buffer and sets P.tile_mask / P.mask_words.  P holds the tree, the staged cameras and options and the work
// decomposition's tiles_x / tiles_y.
int launch_tile_mask(vr_tree* t, LaunchDev& P, cudaStream_t stream);

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
    uint32_t* tile_mask = nullptr;   // tile coverage of the batch march launches on this stream (vr_cull.cu)
    size_t mask_cap = 0;             // its size in words
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
    uint32_t* sigma_grid = nullptr;   // coarse sigma grid (TreeDev::sigma_grid)
    uint4* tab_org = nullptr;         // origin and level of every table (vr_cull.cu), kept for grid rebuilds
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
