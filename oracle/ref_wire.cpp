// ref_wire.cpp -- C-ABI around the UNMODIFIED reference's N3Tree::gen_wireframe (test infrastructure).
//
// Built only where the reference sources exist (oracle/Makefile.wire), into oracle/_ref/, and linked against
// oracle/_ref/libvolrend_ref.so, which holds the reference's own n3tree.cpp.  No reference source is copied.  The
// tree handle is the N3Tree* that ref_tree_open (oracle/ref_harness.cu) returns.
//
//   ref_tree_wireframe -> N3Tree::gen_wireframe (src/n3tree.cpp:365-434), the host walk
#include <algorithm>
#include <chrono>
#include <cstring>
#include <vector>

#include "volrend/n3tree.hpp"

extern "C" {

// gen_wireframe(max_depth) of the opened tree: returns its length in floats and copies up to `cap` of them to
// `out` (out NULL: count only).  *ms (if not NULL) receives the host time of the gen_wireframe call.
long long ref_tree_wireframe(void* tp, int max_depth, float* out, long long cap, double* ms) {
    const volrend::N3Tree& tree = *static_cast<volrend::N3Tree*>(tp);
    const auto t0 = std::chrono::steady_clock::now();
    const std::vector<float> v = tree.gen_wireframe(max_depth);
    const auto t1 = std::chrono::steady_clock::now();
    if (ms) *ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    if (out) memcpy(out, v.data(), sizeof(float) * (size_t)std::min<long long>(cap, (long long)v.size()));
    return (long long)v.size();
}

}  // extern "C"
