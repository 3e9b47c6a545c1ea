// The item source of the discrete env: draw_item delivers the item of draw h.draw_pos and advances it.  The one place the item formulas live:
// the step kernels (pct_discrete.cu) and the item preview (pct_items.cu) both include it.  The preview is a translation unit of its own because a
// new caller inside pct_discrete.cu changed the register allocation of the apply kernels around their calls; `inline` lets both units define it.
#pragma once
#include "pct_common.cuh"
#include "pct_kernels.h"

namespace pct {

__device__ __noinline__ inline void draw_item(const DParams &p, int e, DHdr &h) {
    const uint64_t gid = (uint64_t)(p.env_id_base + e);
    const uint64_t d = (uint64_t)h.draw_pos;
    const double *it;
    if (p.item_mode == 0) {
        it = p.item_set + (rnd_u64(p.seed, gid, d) % (uint64_t)p.n_items) * 3;
        h.next_den = p.setting == 3 ? rnd_density(p.seed, gid, d) : 1.0;
    } else {
        it = p.stream + ((size_t)e * p.stream_len + (size_t)(d % (uint64_t)p.stream_len)) * 4;
        h.next_den = p.setting == 3 ? it[3] : 1.0;
    }
    h.next_box[0] = (int)it[0];
    h.next_box[1] = (int)it[1];
    h.next_box[2] = (int)it[2];
    h.draw_pos++;
}

}  // namespace pct
