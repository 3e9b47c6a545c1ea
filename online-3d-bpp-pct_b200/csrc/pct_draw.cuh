// The item source of each domain (draw_item, draw_item_c) and the discrete env reset that draws from it.  draw_item delivers the item of draw h.draw_pos and advances it;
// reset_space is what a reset does to an env (the auto-reset of the apply kernel and the per-env reset of pct_reset_envs).  The one place
// they live: the step kernels (pct_discrete.cu, pct_continuous.cu), the item / reset kernels (pct_items.cu) and the refill of the buffered
// step (pct_buffer.cu) include it.  The item / reset kernels are a translation unit
// of their own because a new caller inside pct_discrete.cu changed the register allocation of the apply kernels around their calls; `inline`
// lets both units define the functions.
#pragma once
#include "pct_common.cuh"
#include "pct_kernels.h"
#include "pct_stability.cuh"
#include "pct_continuous.cuh"

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

// Space.reset (D:space.py:290-314) + box_creator.reset / generate_box_size (D:bin3D.py:62-65)
__device__ __noinline__ inline void reset_space(DEnvHot *hot, const DParams &p, int e, int lane) {
    if (lane == 0) {
        DHdr &h = hot->h;
        h.n_box = 0; h.n_ems = 1; h.n_leaf = 0; h.flags = 0; h.n_edge = 0; h.n_poly = 0; h.vol_sum = 0; h.ep_len = 0; h.ep_reward = 0;
        hot->ems[0][0] = 0; hot->ems[0][1] = 0; hot->ems[0][2] = 0;
        hot->ems[0][3] = (int16_t)p.W; hot->ems[0][4] = (int16_t)p.L; hot->ems[0][5] = (int16_t)p.H;
        if (p.traj_len > 0 && h.draw_pos % p.traj_len) h.draw_pos += p.traj_len - h.draw_pos % p.traj_len;  // LoadBoxCreator.reset
        draw_item(p, e, h);
    }
    __syncwarp();
}

// the continuous env's item source (C:bin3D.py:103-112): the same contract as draw_item
__device__ __noinline__ inline void draw_item_c(const CParams &p, int e, CHdr &h) {
    const uint64_t gid = (uint64_t)(p.env_id_base + e), d = (uint64_t)h.draw_pos;
    if (p.item_mode == 0 && p.sample_dist) {  // C:bin3D.py:103-112
        auto u01 = [&](uint64_t salt) { return (double)(rnd_u64(p.seed ^ salt, gid, d) >> 11) * (1.0 / 9007199254740992.0); };
        auto r3 = [&](double v) { return ddiv(rint(v * 1000.0), 1000.0); };
        h.next_box[0] = r3(p.sample_a + (p.sample_b - p.sample_a) * u01(0x11));
        h.next_box[1] = r3(p.sample_a + (p.sample_b - p.sample_a) * u01(0x22));
        if (p.setting == 2) h.next_box[2] = r3(p.sample_a + (p.sample_b - p.sample_a) * u01(0x33));
        else {
            const double ch[5] = {0.1, 0.2, 0.3, 0.4, 0.5};
            h.next_box[2] = ch[rnd_u64(p.seed ^ 0x44, gid, d) % 5];
        }
        h.next_den = p.setting == 3 ? rnd_density(p.seed, gid, d) : 1.0;
    } else {
        const double *it = p.item_mode == 0 ? p.item_set + (rnd_u64(p.seed, gid, d) % (uint64_t)p.n_items) * 3
                                            : p.stream + ((size_t)e * p.stream_len + (size_t)(d % (uint64_t)p.stream_len)) * 4;
        h.next_box[0] = it[0]; h.next_box[1] = it[1]; h.next_box[2] = it[2];
        h.next_den = p.setting == 3 ? (p.item_mode == 0 ? rnd_density(p.seed, gid, d) : it[3]) : 1.0;
    }
    h.draw_pos++;
}

}  // namespace pct
