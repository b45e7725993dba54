// ladder_plan.h — the schedule of glava_b200_export_ladder (DESIGN 4.13), host code: every unit of every rung once
// (export_core.h ladder_unit), sorted by the first source row its footprint reads, top-down, then by rung.  The kernel runs
// the units of one entry in this order, so the warps in flight at any moment cover a few source rows of one frame across
// all rungs and the first rung to read a line brings it into L2 for the others.  export.cpp and the host test tier
// (tests/test_export_ladder_core.py) compile this same code.
#ifndef GLAVA_B200_LADDER_PLAN_H
#define GLAVA_B200_LADDER_PLAN_H

#include "export_core.h"

#include <algorithm>
#include <vector>

namespace glb {

// One rung as the schedule sees it: its rectangle (defaults applied), whether it is the whole frame at its own size, and
// whether its scaled items are 4:2:0 row pairs (NV12, I420, P010)
struct LadderGeom { int src_x, src_y, src_w, src_h, out_w, out_h; bool whole, pairs; };

// the whole frame of a w x h renderer at its own size: export_kernel's items
inline bool ladder_whole(int w, int h, const LadderGeom& g) {
    return g.src_x == 0 && g.src_y == 0 && g.src_w == w && g.src_h == h && g.out_w == w && g.out_h == h;
}

// the top-down index of the first source row unit `row` of rung g reads
inline int ladder_first_row(const LadderGeom& g, int row) {
    if (g.whole) return 2 * row;
    return g.src_y + export_span(g.pairs ? 2 * row : row, g.src_h, g.out_h).first;
}

// the units of every rung of a w x h frame, in schedule order
inline std::vector<uint64_t> ladder_schedule(int w, int h, const LadderGeom* rungs, int nrungs) {
    struct Keyed { int first, rung; uint64_t unit; };
    std::vector<Keyed> all;
    for (int r = 0; r < nrungs; ++r) {
        const LadderGeom& g = rungs[r];
        const int rows = g.whole ? (h + 1) >> 1 : g.pairs ? g.out_h >> 1 : g.out_h;
        const int cols = g.whole ? (w + 127) >> 7 : (g.out_w + 31) >> 5;
        for (int row = 0; row < rows; ++row) {
            const int first = ladder_first_row(g, row);
            for (int col = 0; col < cols; ++col) all.push_back({ first, r, ladder_unit(r, row, col) });
        }
    }
    std::stable_sort(all.begin(), all.end(), [](const Keyed& a, const Keyed& b) {
        return a.first != b.first ? a.first < b.first : a.rung < b.rung;
    });
    std::vector<uint64_t> out(all.size());
    for (size_t i = 0; i < all.size(); ++i) out[i] = all[i].unit;
    return out;
}

}  // namespace glb
#endif
