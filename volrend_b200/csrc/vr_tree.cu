// vr_tree.cu -- the device layout of a tree (the job of N3Tree::load_cuda, reference src/cuda/n3tree.cu:9-41):
// pinned upload of the source arrays, re-layout of the child links, node depths, and the wide tables with their
// colour records, which are all the march kernels read.  Declared in include/volrend_b200.h (vr_tree_create*,
// vr_tree_destroy, vr_tree_get_info).
#include <cuda_runtime.h>

#include <cub/device/device_scan.cuh>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "vr_kernels.h"
#include "vr_tree.h"

using namespace vrb;

// ------------------------------------------------------------------------------------ upload
namespace {

// Host -> device copy of a large pageable array at pinned-memory speed: a few worker threads copy
// chunks into process-wide pinned staging buffers and issue the DMA from there (the reference uploads
// with one synchronous pageable cudaMemcpy, src/cuda/n3tree.cu:20-33, ~12 GB/s).
class Uploader {
  public:
    static constexpr int kWorkers = 4;
    static constexpr size_t kChunk = 8u << 20;
    static Uploader& get() { static Uploader u; return u; }
    cudaError_t copy(void* dst, const void* src, size_t bytes) {
        if (bytes < 4 * kChunk || !ensure()) return cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
        std::lock_guard<std::mutex> lk(mu_);
        int dev = 0;
        cudaGetDevice(&dev);
        const size_t n_chunks = (bytes + kChunk - 1) / kChunk;
        std::atomic<int> err{0};
        std::vector<std::thread> th;
        for (int w = 0; w < kWorkers; ++w)
            th.emplace_back([&, w]() {
                cudaSetDevice(dev);
                cudaStream_t st = nullptr;
                cudaEvent_t ev[2] = {nullptr, nullptr};
                if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) { err = 1; return; }
                for (auto& e : ev) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
                int k = 0;
                for (size_t c = (size_t)w; c < n_chunks && !err; c += kWorkers, ++k) {
                    const size_t off = c * kChunk, n = bytes - off < kChunk ? bytes - off : kChunk;
                    unsigned char* stage = stage_[2 * w + (k & 1)];
                    if (k >= 2) cudaEventSynchronize(ev[k & 1]);   // the DMA that last read this buffer is done
                    memcpy(stage, (const unsigned char*)src + off, n);
                    if (cudaMemcpyAsync((unsigned char*)dst + off, stage, n, cudaMemcpyHostToDevice, st) != cudaSuccess) err = 1;
                    cudaEventRecord(ev[k & 1], st);
                }
                if (cudaStreamSynchronize(st) != cudaSuccess) err = 1;
                for (auto& e : ev) cudaEventDestroy(e);
                cudaStreamDestroy(st);
            });
        for (auto& t : th) t.join();
        return err ? cudaErrorUnknown : cudaSuccess;
    }

  private:
    bool ensure() {
        std::lock_guard<std::mutex> lk(mu_);
        if (ready_) return true;
        if (failed_) return false;
        for (int i = 0; i < 2 * kWorkers; ++i)
            if (cudaHostAlloc((void**)&stage_[i], kChunk, cudaHostAllocDefault) != cudaSuccess) {
                cudaGetLastError();
                failed_ = true;
                return false;
            }
        ready_ = true;
        return true;
    }
    std::mutex mu_;
    unsigned char* stage_[2 * kWorkers] = {};
    bool ready_ = false, failed_ = false;
};

}  // namespace

// ------------------------------------------------------------------------------------ re-layout kernels
namespace {

// Source of the fp16 leaf data: the plain [slot][data_dim] array, or a quantised tree
// (scripts/compress_octree.py; CPU decode in src/n3tree.cpp:309-340):
//   data[slot][j + n_retain + k*n_total] = quant_colors[j][quant_map[j][slot]][k]   j < n_quant
//   data[slot][j + k*n_total]            = data_retained[j][slot][k]                j < n_retain
//   data[slot][data_dim-1]               = sigma[slot]
struct LeafSrc {
    const unsigned short* data;      // plain
    const unsigned short* colors;    // quantised
    const unsigned short* qmap;
    const unsigned short* retained;
    const unsigned short* sigma;
    long long n_slots;
    int data_dim, basis_dim, kbd, n_total, n_retain;
};

__device__ __forceinline__ unsigned short leaf_sigma(const LeafSrc& S, long long slot) {
    return S.data ? S.data[(size_t)slot * S.data_dim + (S.data_dim - 1)] : S.sigma[slot];
}

// half c (= channel * kbd + j) of the padded colour record of `slot`
__device__ __forceinline__ unsigned short leaf_half(const LeafSrc& S, long long slot, int c) {
    if (S.kbd <= 1) {  // one coefficient per channel: RGBA -> halfs 0,1,2 ; basis -> k[0], k[bd], k[2bd]
        if (c >= 3) return 0;
        if (S.data) return S.data[(size_t)slot * S.data_dim + (S.kbd < 0 ? c : c * S.basis_dim)];
        const int j = 0, k = c;  // quantised trees are never RGBA
        if (j < S.n_retain) return S.retained[((size_t)j * S.n_slots + slot) * 3 + k];
        return S.colors[((size_t)(j - S.n_retain) * 65536 + S.qmap[(size_t)(j - S.n_retain) * S.n_slots + slot]) * 3 + k];
    }
    if (c >= 3 * S.kbd) return 0;
    if (S.data) return S.data[(size_t)slot * S.data_dim + c];
    const int j = c % S.n_total, k = c / S.n_total;   // kbd == n_total here
    if (j < S.n_retain) return S.retained[((size_t)j * S.n_slots + slot) * 3 + k];
    const int q = j - S.n_retain;
    return S.colors[((size_t)q * 65536 + S.qmap[(size_t)q * S.n_slots + slot]) * 3 + k];
}

// Node word of a link outside [1, capacity): neither a node id (< 2^28) nor a leaf word.  Only an error when the
// depth sweep reaches it -- the reference never follows the links of unreachable nodes.
constexpr uint32_t kBadLink = 0x7fffffffu;

// nodes[i]: absolute child id, leaf bit | sigma, or kBadLink.
__global__ void relayout_nodes_kernel(const int32_t* __restrict__ child, LeafSrc S, uint32_t* __restrict__ nodes,
                                      long long capacity) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S.n_slots) return;
    const int32_t rel = child[i];
    if (rel != 0) {
        const long long tgt = (i >> 3) + rel;
        nodes[i] = (tgt <= 0 || tgt >= capacity) ? kBadLink : (uint32_t)tgt;
    } else {
        nodes[i] = kLeafBit | (uint32_t)leaf_sigma(S, i);
    }
}

// depth[n] of every node by level-synchronous relaxation from the root.  A node that is reached
// twice (two parents, or a cycle) makes the input a DAG, not a tree: rejected, because the table
// builder and the ancestor stacks assume one depth per node.  So is a reached link outside [1, capacity).
__global__ void node_depth_kernel(const uint32_t* __restrict__ nodes, int* __restrict__ depth, long long capacity,
                                  int level, int* __restrict__ flags) {
    const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= capacity || depth[n] != level) return;
#pragma unroll
    for (int s = 0; s < 8; ++s) {
        const uint32_t w = nodes[n * 8 + s];
        if (w == kBadLink) {
            atomicExch(flags, 1);
        } else if (!(w & kLeafBit)) {
            if (atomicCAS(&depth[w], -1, level + 1) != -1) atomicExch(flags + 2, 1);
            flags[1] = 1;
        }
    }
}

// cnt[r]: number of internal nodes whose depth is r modulo kWideLv
__global__ void count_parity_kernel(const int* __restrict__ depth, long long capacity, unsigned long long* __restrict__ cnt) {
    const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int r = (n < capacity && depth[n] >= 0) ? depth[n] % kWideLv : -1;
#pragma unroll
    for (int k = 0; k < kWideLv; ++k) {
        const unsigned int c = __reduce_add_sync(0xffffffffu, r == k ? 1u : 0u);
        if ((threadIdx.x & 31) == 0 && c) atomicAdd(cnt + k, (unsigned long long)c);
    }
}

// a node owns a table when it is the root or its depth d has (d + v) % kWideLv == 0
__global__ void table_flag_kernel(const int* __restrict__ depth, long long capacity, int v, uint32_t* __restrict__ flag) {
    const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= capacity) return;
    const int d = depth[n];
    flag[n] = (d >= 0 && (n == 0 || (d + v) % kWideLv == 0)) ? 1u : 0u;
}

// wide[table * E + e], E = 8^kWideLv: e = ex << 2*LV | ey << LV | ez holds kWideLv octree levels per axis, first level
// in the high bit.  The tree hangs v levels below a virtual root (octant 0 each time), so the root table resolves only
// kWideLv - v real levels: its entries with a non-zero virtual bit are never looked up.
__global__ void build_wide_kernel(const uint32_t* __restrict__ nodes, const int* __restrict__ depth,
                                  const uint32_t* __restrict__ tid, uint32_t* __restrict__ wide,
                                  uint32_t* __restrict__ wslot, long long capacity, int v) {
    constexpr int LV = kWideLv, M = (1 << LV) - 1;
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n = g >> (3 * LV);
    const int e = (int)(g & (kWideEntries - 1));
    if (n >= capacity) return;
    const int d = depth[n];
    if (d < 0 || (n != 0 && (d + v) % LV != 0)) return;   // unreachable, or folded into an ancestor's table
    // leaf entry = kLeafBit | (103 + leaf depth + v) << 23 | sigma: the exponent field of the cube size on the
    // 2^(24-v) position grid (vr_march.cuh)
    const uint32_t ex = (e >> (2 * LV)) & M, ey = (e >> LV) & M, ez = e & M;
    const size_t o = (size_t)tid[n] * kWideEntries + e;
    uint32_t node = (uint32_t)n;
    int dn = d;
    for (int k = (n == 0) ? v : 0; k < LV; ++k) {
        const int sh = LV - 1 - k;
        const uint32_t oct = (((ex >> sh) & 1u) << 2) | (((ey >> sh) & 1u) << 1) | ((ez >> sh) & 1u);
        const uint32_t s = node * 8u + oct;
        const uint32_t w = nodes[s];
        if (w & kLeafBit) {
            wide[o] = kLeafBit | ((uint32_t)(103 + dn + 1 + v) << 23) | (w & 0xffffu);
            wslot[o] = s;
            return;
        }
        node = w;
        ++dn;
    }
    wide[o] = tid[node];
    wslot[o] = 0xffffffffu;
}

// wrecs[entry]: padded colour record of the entry's leaf, straight from the source arrays
// (16-byte chunks; 8-byte records as one chunk).  Entries that are not leaves stay zero.
// wide != nullptr (vr_tree_update_data): also the sigma bits (low 16) of every leaf entry's word, from the same source.
__global__ void build_wrecs_kernel(const uint32_t* __restrict__ wslot, LeafSrc S, unsigned char* __restrict__ wrecs,
                                   long long n_entries, int rec_bytes, uint32_t* __restrict__ wide = nullptr) {
    const int chunks = rec_bytes >= 16 ? rec_bytes / 16 : 1;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long e = gid / chunks;
    const int c = (int)(gid % chunks);
    if (e >= n_entries) return;
    const uint32_t slot = wslot[e];
    const bool leaf = slot != 0xffffffffu;
    if (wide && leaf && c == 0) wide[e] = (wide[e] & 0xffff0000u) | leaf_sigma(S, slot);
    if (rec_bytes == 8) {
        ushort4 v = make_ushort4(0, 0, 0, 0);
        if (leaf) { v.x = leaf_half(S, slot, 0); v.y = leaf_half(S, slot, 1); v.z = leaf_half(S, slot, 2); }
        reinterpret_cast<ushort4*>(wrecs)[e] = v;
        return;
    }
    unsigned short h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (leaf) {
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = leaf_half(S, slot, c * 8 + j);
    }
    uint4 v;
    v.x = h[0] | ((uint32_t)h[1] << 16); v.y = h[2] | ((uint32_t)h[3] << 16);
    v.z = h[4] | ((uint32_t)h[5] << 16); v.w = h[6] | ((uint32_t)h[7] << 16);
    reinterpret_cast<uint4*>(wrecs + (size_t)e * rec_bytes)[c] = v;
}

int kernel_basis(int format, int basis_dim) {
    if (format == VR_FMT_RGBA || basis_dim < 0) return -1;
    // rt_core.cuh:134-160: no switch case matches -> only coefficient 0
    return kbd_built(basis_dim) ? basis_dim : 1;
}
int rec_bytes_for(int kbd) { return kbd <= 1 ? 8 : ((3 * kbd * 2 + 15) / 16) * 16; }

}  // namespace

extern "C" {

void vr_tree_destroy(vr_tree* t) {
    if (!t) return;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(t->device);
    cudaFree(t->nodes); cudaFree(t->extra);
    cudaFree(t->wide); cudaFree(t->wslot); cudaFree(t->wrecs);
    for (auto& kv : t->res) { cudaFree(kv.second.queues); cudaFree(kv.second.cam_ring); cudaFree(kv.second.opt_ring); }
    for (int i = 0; i < vr_tree::HostPath::kRing; ++i) {
        cudaFree(t->host.buf[i]);
        if (t->host.rendered[i]) cudaEventDestroy(t->host.rendered[i]);
        if (t->host.copied[i]) cudaEventDestroy(t->host.copied[i]);
    }
    for (auto st : t->host.sr) if (st) cudaStreamDestroy(st);
    if (t->host.sc) cudaStreamDestroy(t->host.sc);
    cudaSetDevice(prev);
    delete t;
}

static int tree_create_impl(const vr_tree_desc* d, const vr_tree_quant_desc* q, uint32_t create_flags, vr_tree** out) {
    if (!d || !out) return fail(VR_EINVAL, "null argument");
    *out = nullptr;
    if (create_flags & ~(uint32_t)VR_TREE_SLOT_MAP) return fail(VR_EINVAL, "unknown tree flags 0x%x", create_flags);
    if (int rc = need_device(nullptr)) return rc;
    if (d->N != 2) return fail(VR_EUNSUPPORTED, "N=%d: only N=2 octrees are supported (as in the reference)", d->N);
    if (d->capacity < 1 || d->capacity >= (1ll << 28)) return fail(VR_EINVAL, "capacity %lld out of range", (long long)d->capacity);
    if (!d->child || (!q && !d->data)) return fail(VR_EINVAL, "child/data arrays missing");
    if (q) {
        if (!q->quant_colors || !q->quant_map || !q->sigma) return fail(VR_EINVAL, "quantised arrays missing");
        if (q->n_quant < 1 || q->n_retain < 0 || (q->n_retain > 0 && !q->data_retained))
            return fail(VR_EINVAL, "bad quantised basis counts");
        if (d->format == VR_FMT_RGBA || q->n_quant + q->n_retain != d->basis_dim)
            return fail(VR_EINVAL, "codebook and map basis numbers does not match");   // n3tree.cpp:296-299
    }
    if (d->format < VR_FMT_RGBA || d->format > VR_FMT_ASG) return fail(VR_EINVAL, "bad data format %d", d->format);
    const int kbd = kernel_basis(d->format, d->basis_dim);
    if (kbd < 0 ? d->data_dim < 4 : d->data_dim < 3 * d->basis_dim + 1)
        return fail(VR_EINVAL, "data_dim %d too small for format %d basis %d", d->data_dim, d->format, d->basis_dim);
    if ((d->format == VR_FMT_SG || d->format == VR_FMT_ASG) && !d->extra)
        return fail(VR_EINVAL, "SG/ASG trees need extra_data");
    if ((d->format == VR_FMT_SG || d->format == VR_FMT_ASG) && d->basis_dim > VR_BASIS_MAX)
        return fail(VR_EINVAL, "basis_dim %d > %d", d->basis_dim, VR_BASIS_MAX);

    vr_tree* t = new vr_tree();
    struct Guard { vr_tree*& t; bool ok = false; ~Guard() { if (!ok) { vr_tree_destroy(t); t = nullptr; } } } guard{t};
    VR_CUDA(cudaGetDevice(&t->device));
    cudaDeviceProp prop;
    VR_CUDA(cudaGetDeviceProperties(&prop, t->device));
    t->num_sms = prop.multiProcessorCount;
    t->data_dim = d->data_dim;
    const long long n_slots = d->capacity * 8;
    const int rec_bytes = rec_bytes_for(kbd);
    const int TB = 256;
    Uploader& up = Uploader::get();

    // device scratch, freed on every exit path
    std::vector<void*> scratch;
    struct Scratch { std::vector<void*>& v; ~Scratch() { for (void* p : v) cudaFree(p); } } scratch_guard{scratch};
    auto dalloc = [&](void** p, size_t bytes) -> cudaError_t {
        cudaError_t e = cudaMalloc(p, bytes ? bytes : 1);
        if (e == cudaSuccess) scratch.push_back(*p);
        return e;
    };
    auto release = [&](void* p) {
        for (auto& s : scratch) if (s == p) { cudaFree(p); s = nullptr; }
    };

    int32_t* raw_child = nullptr;
    int* flags = nullptr;   // {bad link, changed, node reached twice}
    int* depth = nullptr;
    LeafSrc S{};
    S.n_slots = n_slots; S.data_dim = d->data_dim; S.basis_dim = d->basis_dim; S.kbd = kbd;
    S.n_total = d->basis_dim; S.n_retain = q ? q->n_retain : 0;
    VR_CUDA(dalloc((void**)&raw_child, (size_t)n_slots * 4));
    VR_CUDA(dalloc((void**)&flags, 4 * sizeof(int)));
    VR_CUDA(dalloc((void**)&depth, (size_t)d->capacity * sizeof(int)));
    VR_CUDA(cudaMalloc(&t->nodes, (size_t)n_slots * 4));
    VR_CUDA(up.copy(raw_child, d->child, (size_t)n_slots * 4));
    if (!q) {
        unsigned short* raw = nullptr;
        const size_t data_bytes = (size_t)n_slots * d->data_dim * 2;
        VR_CUDA(dalloc((void**)&raw, data_bytes));
        VR_CUDA(up.copy(raw, d->data, data_bytes));
        S.data = raw;
    } else {
        const size_t cb = (size_t)q->n_quant * 65536 * 3 * 2, mb = (size_t)q->n_quant * n_slots * 2,
                     sb = (size_t)n_slots * 2, rb = (size_t)q->n_retain * n_slots * 3 * 2;
        unsigned short *qc = nullptr, *qm = nullptr, *qs = nullptr, *qr = nullptr;
        VR_CUDA(dalloc((void**)&qc, cb));
        VR_CUDA(dalloc((void**)&qm, mb));
        VR_CUDA(dalloc((void**)&qs, sb));
        VR_CUDA(up.copy(qc, q->quant_colors, cb));
        VR_CUDA(up.copy(qm, q->quant_map, mb));
        VR_CUDA(up.copy(qs, q->sigma, sb));
        if (q->n_retain > 0) {
            VR_CUDA(dalloc((void**)&qr, rb));
            VR_CUDA(up.copy(qr, q->data_retained, rb));
        }
        S.colors = qc; S.qmap = qm; S.sigma = qs; S.retained = qr;
    }
    VR_CUDA(cudaMemset(flags, 0, 4 * sizeof(int)));
    if (d->extra && (d->format == VR_FMT_SG || d->format == VR_FMT_ASG)) {
        const size_t nf = (size_t)d->basis_dim * (d->format == VR_FMT_SG ? 4 : 11);
        VR_CUDA(cudaMalloc(&t->extra, nf * sizeof(float)));
        VR_CUDA(cudaMemcpy(t->extra, d->extra, nf * sizeof(float), cudaMemcpyHostToDevice));
    }
    relayout_nodes_kernel<<<(unsigned)((n_slots + TB - 1) / TB), TB>>>(raw_child, S, t->nodes, d->capacity);
    VR_CUDA(cudaGetLastError());
    release(raw_child);

    // node depths (level-synchronous sweep) -> max leaf depth; validates that the links form a tree
    VR_CUDA(cudaMemset(depth, 0xff, (size_t)d->capacity * sizeof(int)));
    VR_CUDA(cudaMemset(depth, 0, sizeof(int)));
    int max_node_depth = 0;
    int h_flags[3] = {0, 0, 0};
    for (int level = 0;; ++level) {
        if (level >= kMaxTreeDepth) return fail(VR_EUNSUPPORTED, "tree deeper than %d levels (or its child links form a cycle)", kMaxTreeDepth);
        VR_CUDA(cudaMemsetAsync(flags + 1, 0, sizeof(int)));
        node_depth_kernel<<<(unsigned)((d->capacity + TB - 1) / TB), TB>>>(t->nodes, depth, d->capacity, level, flags);
        VR_CUDA(cudaMemcpy(h_flags, flags, sizeof(h_flags), cudaMemcpyDeviceToHost));
        if (h_flags[0]) return fail(VR_EINVAL, "child array has links outside [1, capacity)");
        if (h_flags[2]) return fail(VR_EINVAL, "child array is not a tree: a node is reachable along two paths");
        if (!h_flags[1]) break;
        max_node_depth = level + 1;
    }

    // kWideLv-levels-per-step tables.  Which nodes own one: those whose depth d has (d + v) % kWideLv == 0, plus the
    // root; the v with the fewest tables wins -- with another one every table at the deepest internal level would
    // replicate its 8 leaves 8 (or 64) times (several times more colour-record memory).
    unsigned long long* pcnt = nullptr;
    VR_CUDA(dalloc((void**)&pcnt, 4 * sizeof(unsigned long long)));
    VR_CUDA(cudaMemset(pcnt, 0, 4 * sizeof(unsigned long long)));
    count_parity_kernel<<<(unsigned)((d->capacity + TB - 1) / TB), TB>>>(depth, d->capacity, pcnt);
    unsigned long long h_pcnt[4] = {0, 0, 0, 0};
    VR_CUDA(cudaMemcpy(h_pcnt, pcnt, sizeof(h_pcnt), cudaMemcpyDeviceToHost));
    int wp = 0;
    unsigned long long n_tab64 = ~0ull;
    for (int v = 0; v < kWideLv; ++v) {
        if (max_node_depth + 1 + v > 24) continue;   // leaf depth + v must fit the 24-bit position grid
        const unsigned long long nt = h_pcnt[(kWideLv - v) % kWideLv] + (v ? 1 : 0);
        if (nt + 1 < n_tab64 || n_tab64 == ~0ull) { n_tab64 = nt; wp = v; }
    }
    if (const char* e = getenv("VR_WIDE_PARITY")) {
        const int v = atoi(e);
        if (v >= 0 && v < kWideLv && max_node_depth + 1 + v <= 24) { wp = v; n_tab64 = h_pcnt[(kWideLv - v) % kWideLv] + (v ? 1 : 0); }
    }
    if (n_tab64 * (unsigned long long)kWideEntries >= (1ull << 32)) return fail(VR_EUNSUPPORTED, "too many nodes for the wide tables");
    const uint32_t n_tab = (uint32_t)n_tab64;
    const long long n_entries = (long long)n_tab * kWideEntries;
    {
        uint32_t *flag = nullptr, *tid = nullptr;
        void* tmp = nullptr;
        size_t tmp_bytes = 0;
        VR_CUDA(dalloc((void**)&flag, (size_t)d->capacity * 4));
        VR_CUDA(dalloc((void**)&tid, (size_t)d->capacity * 4));
        table_flag_kernel<<<(unsigned)((d->capacity + TB - 1) / TB), TB>>>(depth, d->capacity, wp, flag);
        VR_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, flag, tid, (int)d->capacity));
        VR_CUDA(dalloc(&tmp, tmp_bytes));
        VR_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, flag, tid, (int)d->capacity));
        VR_CUDA(cudaMalloc(&t->wide, (size_t)n_entries * 4));
        VR_CUDA(cudaMalloc(&t->wslot, (size_t)n_entries * 4));
        const long long work = d->capacity * (long long)kWideEntries;
        build_wide_kernel<<<(unsigned)((work + TB - 1) / TB), TB>>>(t->nodes, depth, tid, t->wide, t->wslot, d->capacity, wp);
        VR_CUDA(cudaGetLastError());
        release(flag); release(tid); release(tmp);
    }
    release(depth);
    {
        const size_t wrec_bytes = (size_t)n_entries * rec_bytes;
        const cudaError_t e = cudaMalloc(&t->wrecs, wrec_bytes);
        if (e != cudaSuccess) {
            char what[128];
            snprintf(what, sizeof(what), "colour records of the wide tables need %.2f GB (%lld entries x %d B)",
                     wrec_bytes / 1e9, n_entries, rec_bytes);
            return cuda_fail(e, what);
        }
        const long long rwork = n_entries * (rec_bytes >= 16 ? rec_bytes / 16 : 1);
        build_wrecs_kernel<<<(unsigned)((rwork + TB - 1) / TB), TB>>>(t->wslot, S, t->wrecs, n_entries, rec_bytes);
        VR_CUDA(cudaGetLastError());
    }
    VR_CUDA(cudaDeviceSynchronize());
    // the march kernels read the tables and the table-indexed records only; the weights pass also the slot map
    cudaFree(t->nodes); t->nodes = nullptr;
    const bool slot_map = (create_flags & VR_TREE_SLOT_MAP) != 0;
    if (!slot_map) { cudaFree(t->wslot); t->wslot = nullptr; }
    t->n_tables = n_tab;
    g_launches += 7;

    TreeDev& D = t->dev;
    D.wide = t->wide; D.wrecs = t->wrecs; D.extra = t->extra;
    for (int i = 0; i < 3; ++i) { D.offset[i] = d->offset[i]; D.scale[i] = d->scale[i]; }
    D.ndc_width = d->use_ndc ? d->ndc_width : -1.f;  // data_spec.hpp:47
    D.ndc_height = d->ndc_height; D.ndc_focal = d->ndc_focal;
    D.N = d->N; D.format = d->format; D.basis_dim = d->basis_dim; D.kbd = kbd;
    D.rec_bytes = rec_bytes; D.max_depth = max_node_depth + 1; D.wide_p = wp; D.wide_entries = (uint32_t)n_entries;
    D.pos_scale = (float)(1u << (24 - wp));
    D.pos_hi = (1.f - 1e-6f) * D.pos_scale;   // exact: a power-of-two multiple of 0x3F7FFFEF
    D.icube_bias = 0x73000000u + ((uint32_t)wp << 23);
    vr_tree_info& I = t->info;
    I.capacity = d->capacity; I.max_depth = D.max_depth; I.rec_bytes = rec_bytes;
    I.node_bytes = n_slots * 4; I.rec_total_bytes = n_slots * (long long)rec_bytes;
    I.top_bytes = 16 * 16 * 16 * 4;   // a dense 16^3 grid of node words
    I.kernel_basis = kbd; I.wide_parity = wp; I.n_tables = n_tab;
    I.wide_bytes = n_entries * 4; I.wrecs_bytes = n_entries * (long long)rec_bytes;
    I.kernel_bytes = I.wide_bytes + I.wrecs_bytes;
    I.device_bytes = I.kernel_bytes + (slot_map ? n_entries * 4 : 0);
    guard.ok = true;
    *out = t;
    return VR_OK;
}

int vr_tree_create_ex(const vr_tree_desc* d, uint32_t flags, vr_tree** out) {
    return tree_create_impl(d, nullptr, flags, out);
}
int vr_tree_create(const vr_tree_desc* d, vr_tree** out) { return vr_tree_create_ex(d, 0, out); }

int vr_tree_create_quantized_ex(const vr_tree_quant_desc* q, uint32_t flags, vr_tree** out) {
    if (!q) return fail(VR_EINVAL, "null argument");
    if (q->base.data) return fail(VR_EINVAL, "quantised descriptor must not carry decoded data");
    return tree_create_impl(&q->base, q, flags, out);
}
int vr_tree_create_quantized(const vr_tree_quant_desc* q, vr_tree** out) { return vr_tree_create_quantized_ex(q, 0, out); }

int vr_tree_update_data(vr_tree* t, const uint16_t* data_dev, void* stream) {
    if (!t) return fail(VR_EINVAL, "null tree");
    if (int rc = need_device(t)) return rc;
    if (int rc = need_slot_map(t, "vr_tree_update_data")) return rc;
    if (!data_dev) return fail(VR_EINVAL, "null data");
    if (int rc = buffer_check(t, data_dev, "data_dev")) return rc;
    LeafSrc S{};
    S.data = data_dev;
    S.n_slots = t->info.capacity * 8; S.data_dim = t->data_dim; S.basis_dim = t->dev.basis_dim; S.kbd = t->dev.kbd;
    const long long n_entries = t->dev.wide_entries;
    const int rec_bytes = t->dev.rec_bytes, TB = 256;
    const long long rwork = n_entries * (rec_bytes >= 16 ? rec_bytes / 16 : 1);
    build_wrecs_kernel<<<(unsigned)((rwork + TB - 1) / TB), TB, 0, (cudaStream_t)stream>>>(t->wslot, S, t->wrecs,
                                                                                            n_entries, rec_bytes, t->wide);
    VR_CUDA(cudaGetLastError());
    g_launches += 1;
    {
        std::lock_guard<std::mutex> lk(t->res_mu);
        ++t->data_gen;
    }
    return VR_OK;
}

int vr_tree_get_info(const vr_tree* t, vr_tree_info* info) {
    if (!t || !info) return fail(VR_EINVAL, "null argument");
    *info = t->info;
    return VR_OK;
}

}  // extern "C"
