// vr_march_q.cuh -- the march kernel with a WARP-SHARED SHADING QUEUE (warp-level compaction of the colour work):
// persistent warps + wide tables (vr_march.cuh) + a ballot/popc-compacted ring of shaded samples per warp.
// Default for single-view launches on trees with 4, 9 or 16 basis functions (launch_renderer, the CLI); batches
// default to the inline-shading kernel of vr_march.cuh (launch_march in vr_kernels_inst.cu has the numbers).
//
// Why (tools/lane_sim.c replays the exact sample sequence of the bench frames on the CPU and counts warp
// instructions per scheduling policy):
//   * with inline shading the 190-instruction colour block of rt_core.cuh:125-165 runs whenever ANY lane of the
//     warp sits on a surface: about a third of the 32 lanes active;
//   * a queue shared by the warp keeps the coherent 4x8 tiles for the traversal and compacts the shading work
//     across lanes AND iterations: nearly all 32 lanes in the colour block, and the 96-byte record fetch is waited
//     for once per 32 shaded samples instead of once per shaded warp-iteration;
//   * the price is ~30 instructions per march iteration (two votes, ring bookkeeping, a predicated body) and
//     12 KB more shared memory per CTA (less L1): a small loss in 200-view batches, where other warps hide the
//     inline block's latency, a win on single frames, where the frame waits for its tail.
//
// How: the colour of a sample never feeds back into the traversal (transmittance, early stop and the
// next position depend on sigma and the cell geometry only, rt_core.cuh:116-120,174-187).  So the
// march loop only appends {record index, weight, owner lane} to a 64-slot ring in shared memory
// (ballot + popc compaction).  Whenever 32 items are pending, ALL lanes shade one item each -- any
// lane can shade any ray's sample because the per-ray basis values are parked in shared memory -- and
// write the three colour terms weight/(1+exp(-dot)) back into the slot.  Each owner then adds its
// terms to its own accumulators in slot order == sample order, so every ray performs exactly the
// additions of rt_core.cuh:163 in the reference's order: bit-identical output.
#pragma once
#include "vr_march.cuh"

namespace vrb {

constexpr int kQSlots = 64;          // ring slots per warp (two 32-item windows)
constexpr int kQSlotBytes = 16;      // {idx, weight, owner, -} in; {r, g, b, -} out

template <int KBD>
struct BasisQ { static constexpr int n = (BasisCount<KBD>::n + 3) / 4; };   // float4 groups per ray

__host__ __device__ inline int wide_levels(int max_depth) {
    const int l = wide_table_levels(max_depth);
    return l < 1 ? 1 : l;
}

constexpr int kParkQ = 3;   // float4 groups of ray constants parked across a drain

// shared memory of one CTA: [ control | parked ray constants | basis values | shading queues | table-id stacks ]
template <int KBD>
__host__ __device__ inline size_t queue_smem_bytes(int max_depth) {
    return 16 /* control words, see kCtrlBytes */ + (size_t)wide_levels(max_depth) * kBlock * 4 + (size_t)kParkQ * kBlock * 16 +
           (size_t)BasisQ<KBD>::n * kBlock * 16 + (size_t)(kBlock / 32) * kQSlots * kQSlotBytes;
}

__device__ __forceinline__ void sts128_a(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void lds128_a(uint32_t addr, uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(addr) : "memory");
}

// One channel of rt_core.cuh:130-163: tmp = B0*k0 (+ s[16..24]) (+ s[9..15]) (+ s[4..8]) + s[1..3], every chain
// s[lo..hi] = fma(B_hi, k_hi, ... fma(B_lo, k_lo, B_{lo+1} * k_{lo+1})).  The basis values of the OWNER ray are
// read from shared memory one float4 group at a time and consumed immediately (4 live values instead of
// 16/25): the chains are independent, so visiting the coefficients in memory order and keeping one partial
// sum per chain performs exactly the reference's operations on exactly its operands.
template <int KBD, typename KF>
__device__ __forceinline__ float channel_dot(KF K, uint32_t bs_owner) {
    static_assert(KBD == 4 || KBD == 9 || KBD == 16 || KBD == 25, "queue kernel: 4, 9, 16 or 25 basis functions");
    float tmp0 = 0.f, s1 = 0.f, s4 = 0.f, s9 = 0.f, s16 = 0.f;
#pragma unroll
    for (int q = 0; q < BasisQ<KBD>::n; ++q) {
        uint32_t v[4];
        lds128_a(bs_owner + (uint32_t)q * (32u * 16u), v[0], v[1], v[2], v[3]);
        auto B = [&](int j) -> float { return __uint_as_float(v[j - 4 * q]); };
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int j = 4 * q + k;
            if (j >= KBD) continue;
            if (j == 0) { tmp0 = __fmul_rn(B(0), K(0)); continue; }
            // chain starts: the reference multiplies element lo+1 first, then fuses element lo
            if (j == 1)  { s1 = __fmaf_rn(B(1), K(1), __fmul_rn(B(2), K(2))); continue; }
            if (j == 4)  { s4 = __fmaf_rn(B(4), K(4), __fmul_rn(B(5), K(5))); continue; }
            if (j == 9)  { s9 = __fmaf_rn(B(9), K(9), __fmul_rn(B(10), K(10))); continue; }
            if (j == 16) { s16 = __fmaf_rn(B(16), K(16), __fmul_rn(B(17), K(17))); continue; }
            if (j == 2 || j == 5 || j == 10 || j == 17) continue;  // consumed by the chain start
            if (j <= 3) s1 = __fmaf_rn(B(j), K(j), s1);
            else if (j <= 8) s4 = __fmaf_rn(B(j), K(j), s4);
            else if (j <= 15) s9 = __fmaf_rn(B(j), K(j), s9);
            else s16 = __fmaf_rn(B(j), K(j), s16);
        }
    }
    float tmp = tmp0;
    if constexpr (KBD >= 25) tmp = __fadd_rn(tmp, s16);
    if constexpr (KBD >= 16) tmp = __fadd_rn(tmp, s9);
    if constexpr (KBD >= 9) tmp = __fadd_rn(tmp, s4);
    tmp = __fadd_rn(tmp, s1);
    return tmp;
}

// All lanes: lane i shades item i of the window at q_win (n items) and replaces it by its three colour
// terms weight / (1 + expf(-dot)) (rt_core.cuh:163).
template <int KBD>
__device__ __forceinline__ void drain_window(uint32_t q_win, uint32_t n, uint32_t bs_warp, const unsigned char* __restrict__ wrecs) {
    const uint32_t lane = threadIdx.x & 31u;
    if (lane < n) {
        const uint32_t slot = q_win + lane * kQSlotBytes;
        uint32_t idx, wbits, owner, pad;
        lds128_a(slot, idx, wbits, owner, pad);
        const unsigned char* rec = rec_addr(wrecs, idx, RecBytes<KBD>::n);
        const uint32_t bs_owner = bs_warp + owner * 16u;
        const float weight = __uint_as_float(wbits);
        float out[3];
        if constexpr (RecWords<KBD>::n <= 24) {
            // whole record in flight at once (6 x LDG.128 for SH16)
            uint32_t w[RecWords<KBD>::n];
            load_rec<KBD>(rec, w);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                auto K = [&](int j) -> float {
                    const int h = c * KBD + j;
                    const uint32_t u = w[h >> 1];
                    return half_bits_to_float((h & 1) ? (u >> 16) : u);
                };
                out[c] = sigmoid_weighted(weight, channel_dot<KBD>(K, bs_owner));
            }
        } else {
            // SH25: 160-byte record, one channel (50 bytes inside four 16-byte chunks) at a time
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                constexpr int kHalfs = KBD;
                const int first = (c * kHalfs * 2) / 16;   // first 16-byte chunk of the channel
                uint32_t w[16];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    uint4 qv;
                    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                                 : "=r"(qv.x), "=r"(qv.y), "=r"(qv.z), "=r"(qv.w) : "l"(rec + 16 * (first + i)));
                    w[4 * i] = qv.x; w[4 * i + 1] = qv.y; w[4 * i + 2] = qv.z; w[4 * i + 3] = qv.w;
                }
                auto K = [&](int j) -> float {
                    const int h = c * kHalfs + j - first * 8;
                    const uint32_t u = w[h >> 1];
                    return half_bits_to_float((h & 1) ? (u >> 16) : u);
                };
                out[c] = sigmoid_weighted(weight, channel_dot<KBD>(K, bs_owner));
            }
        }
        sts128_a(slot, __float_as_uint(out[0]), __float_as_uint(out[1]), __float_as_uint(out[2]), 0u);
    }
    __syncwarp();
}

// shared memory of one CTA: [ 16 B | parked ray constants | basis values | shading queues | table-id stacks ]
constexpr uint32_t kCtrlBytes = 16;

// ---------------------------------------------------------------- the kernel
template <int KBD, bool COUNT, int OUT>
__global__ void __launch_bounds__(kBlock, kMinBlocks) march_queue_kernel(const __grid_constant__ LaunchDev P) {
    extern __shared__ __align__(128) unsigned char smem[];
    constexpr int KQ = BasisQ<KBD>::n;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // every region but the last has a compile-time size, so all addresses are constants + f(threadIdx): nothing but
    // the stack pointer has to stay in a register across the march loop
    const uint32_t smem0 = smem_u32(smem) + kCtrlBytes;
    // ray constants of this thread, parked across a drain: rs[quad][thread]
    const uint32_t rs = smem0 + threadIdx.x * 16u;
    const uint32_t bs0 = smem0 + kParkQ * (kBlock * 16u);
    const uint32_t bs_warp = bs0 + (uint32_t)warp * (KQ * 32u * 16u);
    const uint32_t q_warp = bs0 + (kBlock / 32) * (KQ * 32u * 16u) + (uint32_t)warp * (kQSlots * kQSlotBytes);
    // stack[level][thread]; opaque so that the address stays in one register (see march())
    uint32_t stack_a = bs0 + (kBlock / 32) * (KQ * 32u * 16u + kQSlots * kQSlotBytes) + threadIdx.x * 4u;
    asm volatile("mov.u32 %0, %0;" : "+r"(stack_a));
    uint32_t lt_mask;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(lt_mask));

    pdl_launch_dependents();
    Counts cnt = {0, 0, 0, 0, 0};
    bool dep_done = false;
    if (COUNT || P.cams) {  // instrumented runs and batches (camera ring written by a copy) do not overlap
        pdl_wait_predecessor();
        dep_done = true;
    }
    float step = P.opt.step_size, sthr = P.opt.sigma_thresh;
    // kOutViewOpts: the options of the view of the warp's current work item (read when the item is taken, and again
    // for the pixel write, so that only the loop constants stay live across the march)
    OptDev vopt{};
    const OptDev& opt = OUT == kOutViewOpts ? vopt : P.opt;
    const uint32_t* __restrict__ wide = P.tree.wide;
    const int wp = P.tree.wide_p;

    for (;;) {
        // ------------------------------------------------ acquire work: the next tile
        // Which pixel a lane works on travels as ONE word, lane slot << 26 | tile index, in the spare word of the
        // parked ray constants (rs quad 2): nothing about the pixel is live across the march loop.
        uint32_t init = 0;
        Ray R;
        R.t = 0.f; R.tmax = -1.f;
        bool hit = false;
        float t = __int_as_float(0x7fc00000), T = 1.f, r = 0.f, g = 0.f, b = 0.f;   // NaN: no ray in this lane
        Walk W = {0u, 0u, 0u, kWideDepthBias + 1};   // "previous leaf" of a fresh ray: depth 1
        unsigned long long t_begin = 0;

        const unsigned int item = next_item<false>(P, lane);
        if (item == kNoItem) break;
        {
            int view, tx, ty;
            decode_item<false>(P, item, view, tx, ty);
            const int lx = tx * kTW + (lane % kTW), ly = ty * kTH + (lane / kTW);
            const bool inb = lx < P.w && ly < P.h;
            const CamDev& cam = P.cams ? P.cams[view] : P.cam;
            if constexpr (OUT == kOutViewOpts) {
                vopt = P.opts[view];
                step = vopt.step_size; sthr = vopt.sigma_thresh;
            }
            if (COUNT && P.trace) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_begin));

            const int px = P.x0 + lx, py = P.y0 + frame_row(P, ly);
            float tlim = 1e9f;
            if (P.composite && inb) {  // volrend.cu:92-96,143-146
                if (!dep_done) { pdl_wait_predecessor(); dep_done = true; }  // reads the previous image
                const size_t o = ((size_t)view * P.h + ly) * P.w + lx;
                if (OUT == kOutSurface) {
                    init = surf2Dread<uint32_t>(P.surf, px * 4, py, cudaBoundaryModeZero);
                    if (P.dsurf) tlim = surf2Dread<float>(P.dsurf, px * 4, py, cudaBoundaryModeZero);
                } else {
                    init = reinterpret_cast<const uint32_t*>(P.rgba8)[o];
                    if (P.depth_in) tlim = P.depth_in[o];
                }
            }
            if (inb && P.tree.N > 0) {
                float vd[3];
                hit = ray_geometry(P.tree, opt, cam, px, py, tlim, R, vd, P.tree.pos_scale);
                if (hit) {  // basis values of this ray -> shared memory, bs[q][lane]
                    float B[BasisCount<KBD>::n];
                    eval_basis<KBD>(P.tree, opt, vd, B);
#pragma unroll
                    for (int q = 0; q < KQ; ++q) {
                        float v[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) v[k] = (4 * q + k < BasisCount<KBD>::n) ? B[4 * q + k] : 0.f;
                        sts128_a(bs_warp + ((uint32_t)q * 32u + (uint32_t)lane) * 16u, __float_as_uint(v[0]), __float_as_uint(v[1]),
                                 __float_as_uint(v[2]), __float_as_uint(v[3]));
                    }
                }
            }
            if (COUNT && hit) ++cnt.hit;
            if (hit) {  // the drain needs the registers: the ray constants are reloaded after it (hand-made live-range split)
                sts128_a(rs, __float_as_uint(R.dx), __float_as_uint(R.dy), __float_as_uint(R.dz), __float_as_uint(R.cx));
                sts128_a(rs + kBlock * 16u, __float_as_uint(R.cy), __float_as_uint(R.cz), __float_as_uint(R.ix), __float_as_uint(R.iy));
                sts128_a(rs + 2u * kBlock * 16u, __float_as_uint(R.iz), __float_as_uint(R.tmax), __float_as_uint(R.ds), 0u);
            }
            asm volatile("st.shared.u32 [%0], %1;" :: "r"(rs + 2u * kBlock * 16u + 12u), "r"(((uint32_t)lane << 26) | item) : "memory");
            // Ray state.  A finished ray is encoded in t itself: t >= tmax at a normal end, t = +inf after an
            // early stop (rt_core.cuh:176), so no flag has to be carried through the loop.
            t = hit ? R.t : __int_as_float(0x7fc00000);   // NaN: t < tmax is false, and it is not the early-stop marker
            asm volatile("st.shared.u32 [%0], %1;" :: "r"(stack_a), "r"(0u) : "memory");
        }
        uint32_t mine_cur = 0u, mine_next = 0u;   // slots of the draining / the following window that hold this lane's samples
        uint32_t qhead = 0u, qcount = 0u;         // warp-uniform

        const bool want_colour = !opt.render_depth;
        do {   // march until no ray of the warp is alive
            bool shaded = false;   // this lane produced a sample whose colour has to be evaluated
            uint32_t eidx;
            float weight;
            // (taking 2 or 3 samples per lane between two rounds of votes was measured: slower)
            if (t < R.tmax) {   // rt_core.cuh:108
                float x, y, z;
                uint32_t ux, uy, uz, w;
                int depth;
                sample_pos(R, t, x, y, z, ux, uy, uz, P.tree.pos_hi);
                find_leaf_wide<COUNT>(wide, stack_a, W, ux, uy, uz, w, eidx, depth, cnt, wp);
                if (COUNT) { ++cnt.samples; cnt.child_loads += depth; }
                const float dt = cell_delta_t(R, x, y, z, step, w, P.tree.icube_bias);
                const float sigma = half_bits_to_float(w);
                bool stop = false;
                if (sigma > sthr) {                 // :118
                    const float att = expf_pinned(__fmul_rn(__fmul_rn(-dt, R.ds), sigma));  // :119
                    weight = __fmul_rn(T, __fsub_rn(1.f, att));                               // :120
                    if (COUNT) ++cnt.shaded;
                    if (!want_colour) r = __fmaf_rn(t, weight, r);  // :122-123
                    shaded = want_colour;
                    T = __fmul_rn(T, att);  // :174
                    stop = T < opt.stop_thresh;   // :176
                }
                t = stop ? __int_as_float(0x7f800000) : __fadd_rn(t, dt);        // :187, or the early-stop marker
            }
            const uint32_t bal = __ballot_sync(0xffffffffu, shaded);
            if (bal) {
                const uint32_t rel = qcount + (uint32_t)__popc(bal & lt_mask);   // position behind the ring head, < 64
                if (shaded) {
                    sts128_a(q_warp + ((qhead + rel) & (kQSlots - 1)) * kQSlotBytes, eidx, __float_as_uint(weight), (uint32_t)lane, 0u);
                    const uint32_t bit = 1u << (rel & 31u);
                    if (rel & 32u) mine_next |= bit; else mine_cur |= bit;
                }
                qcount += (uint32_t)__popc(bal);
                if (qcount >= 32u) {
                    __syncwarp();
                    drain_window<KBD>(q_warp + qhead * kQSlotBytes, 32u, bs_warp, P.tree.wrecs);
                    uint32_t m = mine_cur;
                    while (m) {  // this lane's terms, in sample order (rt_core.cuh:163)
                        const uint32_t sl = (uint32_t)__ffs((int)m) - 1u;
                        m &= m - 1u;
                        uint32_t cr, cg, cb, pad;
                        lds128_a(q_warp + (qhead + sl) * kQSlotBytes, cr, cg, cb, pad);
                        r = __fadd_rn(r, __uint_as_float(cr)); g = __fadd_rn(g, __uint_as_float(cg)); b = __fadd_rn(b, __uint_as_float(cb));
                    }
                    __syncwarp();   // every owner has read its terms before a later enqueue may reuse the window (racecheck)
                    mine_cur = mine_next;
                    mine_next = 0u;
                    qhead ^= 32u;
                    qcount -= 32u;
                    {   // ray constants back into registers
                        uint32_t a0, a1, a2, a3;
                        lds128_a(rs, a0, a1, a2, a3);
                        R.dx = __uint_as_float(a0); R.dy = __uint_as_float(a1); R.dz = __uint_as_float(a2); R.cx = __uint_as_float(a3);
                        lds128_a(rs + kBlock * 16u, a0, a1, a2, a3);
                        R.cy = __uint_as_float(a0); R.cz = __uint_as_float(a1); R.ix = __uint_as_float(a2); R.iy = __uint_as_float(a3);
                        lds128_a(rs + 2u * kBlock * 16u, a0, a1, a2, a3);
                        R.iz = __uint_as_float(a0); R.tmax = __uint_as_float(a1); R.ds = __uint_as_float(a2);
                        R.ox = fmaxf(R.ix, 0.f); R.oy = fmaxf(R.iy, 0.f); R.oz = fmaxf(R.iz, 0.f);
                    }
                }
            }
        } while (__ballot_sync(0xffffffffu, t < R.tmax) != 0u);
        const bool stopped = __float_as_uint(t) == 0x7f800000u;
        if (qcount) {  // tile end: the remaining items (all in the window at qhead)
            __syncwarp();
            drain_window<KBD>(q_warp + qhead * kQSlotBytes, qcount, bs_warp, P.tree.wrecs);
            uint32_t m = mine_cur;
            while (m) {
                const uint32_t sl = (uint32_t)__ffs((int)m) - 1u;
                m &= m - 1u;
                uint32_t cr, cg, cb, pad;
                lds128_a(q_warp + (qhead + sl) * kQSlotBytes, cr, cg, cb, pad);
                r = __fadd_rn(r, __uint_as_float(cr)); g = __fadd_rn(g, __uint_as_float(cg)); b = __fadd_rn(b, __uint_as_float(cb));
            }
        }
        __syncwarp();   // every lane is done with the ring and the basis values before the next tile reuses them

        // this lane's pixel
        uint32_t packed;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(packed) : "r"(rs + 2u * kBlock * 16u + 12u) : "memory");
        int view, tx, ty;
        decode_item<false>(P, packed & 0x3ffffffu, view, tx, ty);
        const int lx = tx * kTW + (int)((packed >> 26) % kTW), ly = ty * kTH + (int)((packed >> 26) / kTW);
        hit = __float_as_uint(t) != 0x7fc00000u;   // lanes without a ray kept the plain NaN
        if (lx < P.w && ly < P.h) {
            if constexpr (OUT == kOutViewOpts) vopt = P.opts[view];
            const int px = P.x0 + lx, py = P.y0 + frame_row(P, ly);
            float out[4] = {0.f, 0.f, 0.f, 0.f};
            if (hit) {
                if (opt.render_depth) r = g = b = fminf(r * 0.3f, 1.0f);  // :177-179,189-191
                if (stopped) {  // :181-184
                    const float sc = __frcp_rn(__fsub_rn(1.f, T));
                    out[0] = __fmul_rn(r, sc); out[1] = __fmul_rn(g, sc); out[2] = __fmul_rn(b, sc); out[3] = 1.f;
                } else {
                    out[0] = r; out[1] = g; out[2] = b;
                    out[3] = opt.render_depth ? 1.f : __fsub_rn(1.f, T);
                }
            } else if (P.tree.N > 0 && opt.render_depth) {
                out[3] = 1.f;  // rt_core.cuh:90-91
            }
            const float nalpha = __fsub_rn(1.f, out[3]);
            if (!P.composite) {
                const float remain = __fmul_rn(nalpha, opt.background_brightness);
                out[0] = __fadd_rn(remain, out[0]); out[1] = __fadd_rn(remain, out[1]); out[2] = __fadd_rn(remain, out[2]);
            } else {
                out[0] += (float)(init & 0xffu) / 255.f * nalpha;
                out[1] += (float)((init >> 8) & 0xffu) / 255.f * nalpha;
                out[2] += (float)((init >> 16) & 0xffu) / 255.f * nalpha;
            }
            const uint32_t q = quantise(out);
            if (!dep_done) { pdl_wait_predecessor(); dep_done = true; }  // first write of this thread
            const size_t o = ((size_t)view * P.h + ly) * P.w + lx;
            if (OUT == kOutSurface) {
                surf2Dwrite(q, P.surf, px * 4, py, cudaBoundaryModeZero);
            } else {
                if (P.rgba8) reinterpret_cast<uint32_t*>(P.rgba8)[o] = q;
            }
            if (P.rgbaf) P.rgbaf[o] = make_float4(out[0], out[1], out[2], out[3]);
        }
        __syncwarp();
        if (COUNT && P.trace && lane == 0) {
            unsigned long long t_end;
            unsigned int smid;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end));
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            P.trace[4 * (size_t)item + 0] = t_begin;
            P.trace[4 * (size_t)item + 1] = t_end;
            P.trace[4 * (size_t)item + 2] = smid;
            P.trace[4 * (size_t)item + 3] = blockIdx.x * (kBlock / 32) + (threadIdx.x >> 5);
        }
    }
    if (!dep_done) pdl_wait_predecessor();
    if (COUNT) flush_counts(cnt, P.counters);
    rearm_queue<false>(P);
}

}  // namespace vrb
