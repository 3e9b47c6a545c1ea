/* pct_b200 — C ABI of the H100-native batched PCT environment (drop-in boundary).
 *
 * The reference (alexfrom0815/Online-3D-BPP-PCT @ 5e088f2) has no native interface: its
 * environment is a Python gym.Env (pct_envs/PctDiscrete0/bin3D.py:8-188,
 * pct_envs/PctContinuous0/bin3D.py:8-207) fanned out over forked workers by
 * wrapper/shmem_vec_env.py:20-156.  This header is what a ctypes binding of that path binds
 * instead (see INTEGRATION.md): every entry point names the reference interface it replaces.
 *
 * Conventions
 *   - plain C types only; device pointers are raw CUDA device addresses (e.g. tensor.data_ptr()),
 *     `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *   - every function returns 0 on success or a negative pct_status; pct_last_error() gives text.
 *   - the library owns the per-environment state; the caller owns action / observation / reward /
 *     done / info buffers.  No host synchronisation happens inside pct_reset / pct_step /
 *     pct_policy_random: they only enqueue work on `stream` (CUDA-graph capturable).
 *   - one host thread per handle.
 *
 * Observation layout (identical to D:bin3D.py:86-93 after the float32 cast of envs.py:168,180):
 *   row-major (internal_node_holder + leaf_node_holder + 1, 9)
 *   rows [0, NB)        placed boxes  [x1,y1,z1,x2,y2,z2,density,0,valid]   (row 0 col 8 is always 1)
 *   rows [NB, NB+NL)    leaf nodes    [x1,y1,z1,x2,y2,BIN_H,0,0,valid]
 *   row  NB+NL          next item     [density,0,0,d0<=d1<=d2,0,0,1]
 */
#ifndef PCT_B200_H
#define PCT_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pct_env_batch *pct_handle;

enum pct_status {
    PCT_OK = 0,
    PCT_ERR_INVALID = -1,   /* bad argument / unsupported configuration            */
    PCT_ERR_CUDA = -2,      /* CUDA runtime error (text in pct_last_error)          */
    PCT_ERR_NO_DEVICE = -3, /* no usable sm_90 device: the library has NO CPU fallback */
    PCT_ERR_STATE = -4      /* call sequence error (e.g. step before reset)         */
};

enum pct_domain { PCT_DISCRETE = 0, PCT_CONTINUOUS = 1 };
enum pct_obs_dtype { PCT_F32 = 0, PCT_F64 = 1 };
enum pct_lnes { PCT_LNES_EMS = 0, PCT_LNES_EV = 1, PCT_LNES_EP = 2, PCT_LNES_CP = 3, PCT_LNES_FC = 4 };
/* heuristic baselines of the reference (heuristic.py): LASH :138-226, OnlineBPH :364-424, BR :500-577, MACS :11-131,
 * DBL :431-493, heightmap_min :232-293, random :300-357 */
enum pct_heuristic {
    PCT_H_LSAH = 0, PCT_H_ONLINEBPH = 1, PCT_H_BR = 2, PCT_H_MACS = 3, /* placements taken from the EMS list   */
    PCT_H_DBL = 4, PCT_H_HM = 5, PCT_H_RANDOM = 6                      /* placements taken from the (lx, ly) grid */
};
enum pct_item_mode {
    PCT_ITEMS_RANDOM = 0, /* uniform over item_set with the counter-based generator (RandomBoxCreator, */
                          /*   D:binCreator.py:24-39); continuous + sample_from_distribution: C:bin3D.py:103-115 */
    PCT_ITEMS_STREAM = 1  /* caller-supplied per-env draw sequence (pct_set_item_stream)              */
};

/* Per-environment flag bits reported in pct_step_info.flags (sticky until the env resets). */
enum pct_env_flags {
    PCT_FLAG_BOX_OVERFLOW = 1,      /* more than internal_node_holder boxes (IndexError in D:space.py:385) */
    PCT_FLAG_BAD_ACTION = 2,        /* the reference raises on this action: a leaf row that does not match the item (ValueError in
                                       D:bin3D.py:144-145), or, discrete, a footprint whose slice plain[lx:lx+x, ly:ly+y] is empty under
                                       Python slice rules (np.max of an empty array in D:space.py:354-355; e.g. lx >= max(W, L), or
                                       plain[-1:1]).  The episode ends as for any failed placement, with the same counter and ratio */
    PCT_FLAG_EMS_OVERFLOW = 4,      /* EMS list exceeded the fixed capacity                                */
    PCT_FLAG_CAND_OVERFLOW = 8,     /* candidate set exceeded the fixed capacity                           */
    PCT_FLAG_EDGE_OVERFLOW = 16,    /* support-edge pool exceeded the fixed capacity                       */
    PCT_FLAG_SUPPORT_OVERFLOW = 32, /* more supports under one box than the stability routine handles      */
    PCT_FLAG_SYNC_TIMEOUT = 64,     /* internal: a kernel gave up waiting for the previous stage of this env */
    PCT_FLAG_BAD_SNAPSHOT = 128     /* pct_restore was given a record of another configuration; the env was left as it was   */
};

/* Constructor arguments = the kwargs of PackingDiscrete / PackingContinuous.__init__
 * (D:bin3D.py:9-15, C:bin3D.py:9-17) forwarded by envs.make_env (envs.py:33-47). */
typedef struct pct_config {
    int32_t domain;               /* pct_domain                                                   */
    int32_t setting;              /* 1, 2 or 3                                                    */
    double container_size[3];     /* W, L, H (integers for the discrete domain)                   */
    int32_t internal_node_holder; /* <= 80 in this build                                          */
    int32_t leaf_node_holder;     /* <= 64 in this build                                          */
    int32_t obs_dtype;            /* pct_obs_dtype: float32 (VecPyTorch contract) or float64      */
    int32_t item_mode;            /* pct_item_mode                                                */
    double size_minimum;          /* np.min(item_set) (D:bin3D.py:23) / sample_left_bound (C:bin3D.py:26) */
    int32_t sample_from_distribution; /* continuous only (C:bin3D.py:14)                          */
    double sample_left_bound, sample_right_bound;
    uint64_t seed;                /* item generator seed (PCT_ITEMS_RANDOM)                       */
    int64_t env_id_base;          /* global index of env 0 of this handle (multi-GPU sharding:    */
                                  /*   per-env streams depend on the GLOBAL index only)           */
    int32_t no_auto_reset;        /* 0: ShmemVecEnv worker semantics (finished envs are reset inside the step,   */
                                  /*    wrapper/shmem_vec_env.py:141-142); 1: plain gym.Env semantics (the       */
                                  /*    terminal observation is returned, the caller resets; D:bin3D.py:160-165) */
    int32_t lnes;                 /* leaf-node expansion scheme (D:bin3D.py:101-112): pct_lnes, 0 = EMS (reference default) */
    int32_t shuffle;              /* `shuffle` kwarg (D:bin3D.py:114-115, C:bin3D.py:126-127; tools.py:136 defaults it to True for training): the   */
                                  /*   ordered candidate list is permuted before the feasibility tests and the leaf cap.  The reference draws from  */
                                  /*   the global numpy RNG (no parity definition); here the permutation is the stable argsort of counter-based     */
                                  /*   keys rnd_u64(seed ^ 0x5AFE5EED, global env id, draws << 16 | i) — uniform, reproducible, independent of the  */
                                  /*   sharding — and the oracle (test infrastructure) implements the same definition.                              */
} pct_config;

/* Terminal-step info (the dict built at D:bin3D.py:163-164 plus what Monitor adds, wrapper/monitor.py:58-77) */
typedef struct pct_step_info {
    int32_t counter;    /* len(space.boxes)                                      */
    int32_t flags;      /* pct_env_flags                                         */
    float ratio;        /* space.get_ratio()  (valid when done)                  */
    float ep_reward;    /* sum of rewards of the finished episode (Monitor 'r')  */
    int32_t ep_len;     /* number of steps of the finished episode (Monitor 'l') */
    int32_t n_leaf;     /* number of valid leaf rows in the new observation      */
    int32_t n_cand;     /* number of candidate placements generated (before the feasibility test) */
    int32_t n_ems;      /* EMS count after the step                              */
} pct_step_info;

/* Host-side dump of one environment (parity tests; replaces poking at env.space.* in Python). */
typedef struct pct_state_dump {
    int32_t n_boxes, n_ems, n_leaf, flags;
    int64_t draw_pos;
    double next_box[3];
    double next_den;
    double boxes[80][7]; /* lx,ly,lz,hx,hy,hz,density */
    double ems[256][6];
} pct_state_dump;

/* Host-side dump of the support graph one environment carries from step to step in the stability settings (parity tests): what the
 * real placements' stability descents wrote and every later feasibility walk reads.  Slot-independent: box indices are placement
 * order, list positions are gone.  Box index n_box stands for the box of a FAILED real placement (its loads stay on its supports
 * until the env resets, as the reference's up_edges keep them).
 *   supports of placed box u : sup[sup_off[u] .. sup_off[u+1])                 (stored order = scan order at its placement)
 *   loads resting on box t   : rows load_off[t] .. load_off[t+1]              (insertion order of the reference's up_edges dict)
 *     load_upper = the box the load comes from, load = centre x, y, z and mass as the read-only walks read them,
 *     load_alias = 1: the entry is the upper box's own stack object (alias mode only, else 0)
 *   stored support polygon of box u : poly[poly_off[u] .. poly_off[u+1]) (shrunk hull vertices; only boxes with >= 2 supports store
 *     one, none when the polygon pool had no room), poly_pos[u] = its position in the pool; with exactly two supports
 *     has_split[u] = 1 and split[u] = the stored split direction
 *   own_stack[u] : the box's own stack (centre x, y, z, mass), alias mode only; defined for boxes with a support or a load
 *   alias_stale : alias bits at or beyond n_edge (left by earlier episodes; every new edge rewrites its bit) */
typedef struct pct_support_graph {
    int32_t n_box, n_edge, n_poly, alias;
    int32_t alias_stale, pad_;
    int32_t sup_off[82], load_off[82], poly_off[82], poly_pos[82], has_split[82];
    int32_t sup[256], load_upper[256], load_alias[256];
    double load[256][4];
    double poly[256][2];
    double split[82][2];
    double own_stack[82][4];
} pct_support_graph;

/* gym.make('PctDiscrete-v0' | 'PctContinuous-v0', **kwargs) x n_envs   (envs.py:84-108, tools.py:232-240) */
int pct_create(const pct_config *cfg, int32_t n_envs, int32_t device, pct_handle *out);
/* VecEnv.close()  (wrapper/vec_env.py:93-99) */
void pct_destroy(pct_handle h);
/* text of the last error on this handle (NULL handle: last pct_create error) */
const char *pct_last_error(pct_handle h);

/* item_set kwarg (givenData.py:4-14): host array (n,3) of item sizes used by PCT_ITEMS_RANDOM */
int pct_set_item_set(pct_handle h, const double *items_xyz, int32_t n_items);
/* replaces box_creator (D:binCreator.py): host array (n_envs, len, 4) of (x,y,z,density) draws per env,
 * consumed one per reset and one per successful placement, cyclically. Switches the handle to PCT_ITEMS_STREAM. */
int pct_set_item_stream(pct_handle h, const double *items_xyzd, int32_t len);
/* LoadBoxCreator episodes (D:binCreator.py:41-72): the stream is a sequence of fixed-length trajectories and every
 * reset jumps to the start of the next one (0 = plain continuous stream, the RandomBoxCreator discipline). */
int pct_set_trajectory_length(pct_handle h, int32_t traj_len);

/* VecEnv.reset()  (wrapper/shmem_vec_env.py:61-68 -> D:bin3D.py:61-67): resets every env, writes d_obs
 * (n_envs x obs_len elements of cfg.obs_dtype). */
int pct_reset(pct_handle h, void *d_obs, void *stream);

/* VecEnv.step_async + step_wait  (wrapper/shmem_vec_env.py:70-81,139-143 -> D:bin3D.py:151-188):
 * applies one action per env, auto-resets finished envs (the returned observation of a finished env is
 * its reset observation; reward/done/info are the terminal ones).
 *   d_actions  : n_envs x 9 leaf rows (float32 if action_f64==0 else float64), or NULL
 *   d_leaf_idx : n_envs int32 indices into the previous observation's leaf rows (fast path), or NULL;
 *                an index >= the env's n_leaf, and any NEGATIVE index (no Python-style wrap to the last rows), selects the all-zero
 *                row, which places the item unrotated at (0, 0).  Exactly one of the two is non-NULL.
 *   d_reward   : n_envs float32;  d_done: n_envs uint8;  d_info: n_envs pct_step_info (may be NULL)
 * Observation buffer contract (delta rows, default; PCT_B200_OBS_DELTA=0 restores full rewrites): 75 % of the (internal + leaf + 1) x 9
 * observation is zero padding and the internal-node rows are append-only within an episode, so when a call receives the SAME d_obs pointer
 * as the previous reset / step of this handle, only the rows that can have changed are rewritten (the rows below max(rows now, rows the
 * buffer may hold non-zero) and the item row).  A caller that hands the same buffer to consecutive calls must therefore not modify it in
 * between (reading is fine); a caller that alternates buffers, or passes a fresh one, always gets every row written.  Both domains. */
int pct_step(pct_handle h, const void *d_actions, int32_t action_f64, const int32_t *d_leaf_idx, void *d_obs,
             float *d_reward, uint8_t *d_done, pct_step_info *d_info, void *stream);

/* Same call with HOST buffers (what the reference's VecEnv.step exchanges over its pipes): copies actions host->device, steps, delivers
 * obs / reward / done / info to the host, synchronises.  When h_obs is pinned (cudaHostAlloc / cudaHostRegister, i.e. mapped under UVA) the
 * emit kernel writes the observation rows STRAIGHT into it over PCIe (zero-copy, default; PCT_B200_HOST_ZEROCOPY=0 or an unpinned buffer:
 * staged device buffer + pipelined copies); the buffer contract of pct_step applies to h_obs in that mode. */
int pct_step_host(pct_handle h, const void *h_actions, int32_t action_f64, const int32_t *h_leaf_idx, void *h_obs,
                  float *h_reward, uint8_t *h_done, pct_step_info *h_info);
int pct_reset_host(pct_handle h, void *h_obs);

/* Uniform-random choice among the valid leaf rows of each env (the synthetic policy of SURVEY.md §8(d)):
 * d_leaf_idx[e] = rnd(seed, env_id_base+e, t) % n_leaf[e]  (0 when there is no valid leaf). */
int pct_policy_random(pct_handle h, int32_t *d_leaf_idx, uint64_t seed, int64_t t, void *stream);
/* same, with the step counter read from device memory (*d_t) at execution time: lets a captured CUDA graph of
 * policy -> step draw fresh actions on every replay (the caller increments *d_t inside the graph) */
int pct_policy_random_dev(pct_handle h, int32_t *d_leaf_idx, uint64_t seed, const int64_t *d_t, void *stream);

/* Heuristic baselines, batched (discrete domain).  For every env: the placement the baseline `heuristic` (enum
 * pct_heuristic) selects for the env's current item, written as an action row d_rows[e] = [lx, ly, 0, lx+x, ly+y, 0, 0, 0, 1]
 * (float32, N x 9) that pct_step(d_actions = d_rows, action_f64 = 0) applies; where the baseline finds no feasible
 * placement (the reference then ends the episode without stepping, e.g. heuristic.py:223-225) the row is
 * [1,0,0,1,0,0,0,0,1], which no item matches, so pct_step ends the episode (PCT_FLAG_BAD_ACTION is set in its info).
 * Replaces the per-env Python loops over Space.drop_box_virtual (D:space.py:393-433).  LSAH keeps its running footprint
 * per env inside the handle.  PCT_H_RANDOM draws with rnd(seed, env_id_base+e, t).  PCT_H_BR needs pct_set_item_set.
 * Every baseline runs on every discrete container pct_create accepts (sides up to 255); PCT_H_RANDOM chooses among all
 * feasible grid placements at any size.  The call only enqueues one kernel, so it can be captured in a CUDA graph. */
int pct_heuristic_actions(pct_handle h, int32_t heuristic, float *d_rows, uint64_t seed, int64_t t, void *stream);
/* Same for the CONTINUOUS domain, where tools.py:217-218 allows PCT_H_LSAH, PCT_H_ONLINEBPH and PCT_H_BR only (heuristic.py
 * LASH :138-226, OnlineBPH :364-424, BR :500-577 over pct_envs.PctContinuous0): float64 rows (N x 9) for
 * pct_step(d_actions = d_rows, action_f64 = 1).  "No feasible placement" is the row [W+1,0,0,W+1,0,0,0,0,1]: the continuous
 * LeafNode2Action (C:bin3D.py:151-167) never raises, Space.drop_box rejects the position (C:space.py:336) and the episode ends.
 * Item sizes must carry <= 6 decimals (the reference's generators round to 3, C:bin3D.py:106-111), so that the
 * round(xe - xs, 6) of LeafNode2Action returns the chosen orientation's sizes exactly. */
int pct_heuristic_actions_f64(pct_handle h, int32_t heuristic, double *d_rows, void *stream);
/* Space.drop_box_virtual(dims, (lx, ly), False, density, setting, returnH / returnMap) for ONE env (D:space.py:393-433): what
 * the reference's heuristic.py calls on `env.space`; synchronous.  height_map: W*L int32 (row-major, after the virtual
 * placement — Space.update_height_graph on a copy) or NULL.  Container sides <= 32 (PCT_ERR_INVALID otherwise): for larger
 * bins, pct_query_placements and pct_height_maps answer the same questions without a size limit. */
int pct_query_placement(pct_handle h, int32_t env, const int32_t dims[3], int32_t lx, int32_t ly, double density,
                        int32_t *feasible, int32_t *rest_height, int32_t *height_map);

/* Space.drop_box_virtual(dims, (lx, ly), False, density, setting, returnH=True) of the CONTINUOUS env (C:space.py:380-425) for
 * ONE env; synchronous.  rest_height is interSect2D's max_h (C:space.py:391). */
int pct_query_placement_f64(pct_handle h, int32_t env, const double dims[3], double lx, double ly, double density,
                            int32_t *feasible, double *rest_height);

/* Batched placement queries: Space.drop_box_virtual(dims, (lx, ly), False, density, setting, returnH=True) (D:space.py:393-433,
 * C:space.py:380-425) for many placements of many envs — the primitive for placement rules of one's own (a heuristic, a learned critic
 * over candidate placements, a search on branched envs).  Row r asks k placements of env d_env[r] (d_env NULL: env r).
 *   d_q        : n x k x 5 placements [x, y, z, lx, ly]; x, y, z are the oriented sizes (int32 discrete / float64 continuous)
 *   d_density  : n x k densities, or NULL = each env's current item density (what the facades' drop_box_virtual passes)
 *   d_feasible : n x k uint8;  d_rest_height: n x k int32 / float64 (either output may be NULL)
 * Every answer equals what pct_query_placement(_f64) returns for the same env and inputs, bit for bit, degenerate inputs included: a
 * discrete position outside [0, W) x [0, L) or a zero x / y is infeasible with rest height 0; a footprint that sticks out of the
 * container is infeasible with its rest height still reported; the continuous bounds carry the reference's 1e-6 tolerances.
 * Read-only: env state, sticky flags, the delta-row bookkeeping and the LSAH footprint are untouched (capacity flags of the stability
 * test are not reported), so a step after a query behaves exactly as without it.  Enqueue only: no host synchronisation, no
 * allocation (CUDA-graph capturable).  The env indices of one call must be distinct (caller's contract, as for pct_restore: the
 * stability test of an env uses that env's scratch); a row whose index is outside [0, n_envs) gets feasible 0 and rest height 0.
 * k has no cap, and no container limit applies beyond pct_create's.  n == 0 or k == 0: no-op.  Errors: PCT_ERR_STATE before
 * pct_reset; PCT_ERR_INVALID for the other domain, n < 0, k < 0 or n * k > INT32_MAX. */
int pct_query_placements(pct_handle h, const int32_t *d_env, int32_t n, int32_t k, const int32_t *d_q, const double *d_density,
                         uint8_t *d_feasible, int32_t *d_rest_height, void *stream);   /* discrete   */
int pct_query_placements_f64(pct_handle h, const int32_t *d_env, int32_t n, int32_t k, const double *d_q, const double *d_density,
                             uint8_t *d_feasible, double *d_rest_height, void *stream); /* continuous */
/* Space.plain[:W, :L] (D:space.py:278, 317-326), the height map, of envs d_env[0..n) (d_env NULL: 0..n-1) -> d_out, n x W x L int32
 * (row-major).  Discrete only: the continuous Space has no height map.  An index outside [0, n_envs) gives a zero map.  Same
 * enqueue-only, read-only and error contract as pct_query_placements; no container side limit. */
int pct_height_maps(pct_handle h, const int32_t *d_env, int32_t n, int32_t *d_out, void *stream);

/* Item preview and item override: control over WHICH item an env packs, for lookahead ("online packing with lookahead": the agent
 * knows the next k items) and buffer packing (the agent picks one of B buffered items, then places it).  Both calls only enqueue
 * kernels on `stream`: no host synchronisation, no allocation (CUDA-graph capturable).  Errors: PCT_ERR_STATE before pct_reset;
 * PCT_ERR_INVALID for n < 0, k < 1 or n * k > INT32_MAX.  n == 0: no-op.  The envs named in one call must be distinct (caller's
 * contract, as for pct_restore).
 *
 * BoxCreator.preview(k) (D:binCreator.py:15-18), batched and read-only: d_out[i][0] = env d_env[i]'s CURRENT item (next_box,
 * next_den); d_out[i][j >= 1] = the item its source delivers at draw draw_pos + j - 1 (d_env NULL: env i).  n x k x 4 float64
 * [x, y, z, density]; the density is 1 outside setting 3, as the draws deliver it.  Every item mode: the random item set (setting 3
 * densities included), continuous sample_from_distribution, and per-env streams, which wrap cyclically.  The preview lists raw
 * consecutive draws: a reset in between (the jump to the next trajectory of pct_set_trajectory_length) makes the entries past it
 * stale.  A row whose index is outside [0, n_envs) is all zeros. */
int pct_preview_items(pct_handle h, const int32_t *d_env, int32_t n, int32_t k, double *d_out, void *stream);

/* env d_env[i] <- item i as its current item (d_env NULL: env i): `env.next_box = item; env.next_den = density` followed by the leaf
 * expansion of cur_observation (D:bin3D.py:70-93, without gen_next_box), whose observation rows are written to d_obs (n_envs x obs_len,
 * the layout and delta-row buffer contract of pct_step).
 *   d_items  : n x 3 sizes, int32 (discrete; clamped to [0, 255], the range of a container side) / float64 (continuous)
 *   d_density: n densities, or NULL = keep each env's current density (the draws deliver 1 outside setting 3)
 *   d_info   : n_envs pct_step_info records (may be NULL): counter, sticky flags, n_leaf, n_cand, n_ems; ratio / ep_reward / ep_len 0.
 * No draw is consumed (draw_pos is unchanged).  The set item stays the env's current item until a step places it or the env
 * resets: the next step's reward, LeafNode2Action check and placement use it, a snapshot records it, and after a successful step
 * the env continues with its source's next draw — as in the reference, where `env.next_box = X` then `step` pops the creator's head,
 * not X (D:bin3D.py:180-182).  One difference: after a FAILED step with no_auto_reset the reference's terminal observation
 * re-reads the creator's head (cur_observation -> gen_next_box = preview(1)[0]); here the env keeps the set item, so the terminal
 * observation's item row and leaf rows are those of the set item (what pct_set_items wrote for it).
 * Whole-batch re-expansion: EVERY env of the handle is re-expanded, not only the listed ones, and d_obs receives every env's rows.
 * Envs not listed keep their item and come out bit-identical (same leaves, same rows: the shuffle keys depend on draw_pos only).  So
 * the call costs about one pct_step minus its apply kernel, whatever n is; branch the envs to search over into a handle of their
 * own (pct_snapshot / pct_restore) to pay for those alone.  Capacity flags raised by the new item's expansion are sticky as usual:
 * reported in d_info and by the next step. */
int pct_set_items(pct_handle h, const int32_t *d_env, int32_t n, const void *d_items, const double *d_density, void *d_obs,
                  pct_step_info *d_info, void *stream);

/* Leaf expansion of items the envs are not holding, read-only: for a buffer policy (the PCT tree of a buffered state holds the leaves of
 * each of the B buffered items; choosing a leaf chooses the item) and for lookahead over candidate future items.
 * Row r expands k items on env d_env[r] (d_env NULL: env r) in its current state:
 *   d_items  : n x k x 3 sizes, int32 (discrete; clamped to [0, 255] as pct_set_items clamps) / float64 (continuous)
 *   d_density: n x k densities, or NULL = each env's current item density
 *   d_leaves : n x k x leaf_node_holder x 9, the handle's observation dtype.  Entry (r, j) holds the leaf rows get_possible_position()
 *              (D:bin3D.py:100-136, C:bin3D.py) produces for item d_items[r][j]: the first leaf_node_holder feasible candidates in reference
 *              order as [xs, ys, zs, xe, ye, H, 0, 0, 1], zero rows after the last.  These are the bytes of the leaf rows that pct_set_items
 *              writes into the observation for that item on that env (same cast, LNES scheme and keyed shuffle, whose keys depend on
 *              (seed, global env id, draw_pos) only), so leaf l of the expansion is leaf l of pct_set_items(item) and of the step after it.
 *   d_info   : n x k pct_step_info records, or NULL: the record pct_set_items would write for that env and item: counter, the env's sticky
 *              flags ORed with the capacity flags this expansion raised, n_leaf, n_cand, n_ems; ratio / ep_reward / ep_len 0.
 * Read-only: no header field, leaf list, delta-row state or observation row of any env is written, and a flag raised by an expansion goes to
 * its own record only, so a step after the call behaves exactly as without it.  The call uses the per-env scratch that every step rewrites
 * before reading it (candidate list, generator and shuffle scratch, the stability test's large-case scratch).  The envs of one call must be
 * distinct (caller's contract, not checked: that scratch is per env).  An item that fits nowhere (the [100, 100, 100] sentinel) gets zero
 * leaves; a row whose index is outside [0, n_envs) gets zero rows and zero records.  Enqueue only: no host synchronisation, no allocation
 * (CUDA-graph capturable).  n == 0: no-op.  Errors: PCT_ERR_STATE before pct_reset; PCT_ERR_INVALID for n < 0, k < 1 or
 * n * k * leaf_node_holder * 9 > INT32_MAX. */
int pct_expand_items(pct_handle h, const int32_t *d_env, int32_t n, int32_t k, const void *d_items, const double *d_density, void *d_leaves,
                     pct_step_info *d_info, void *stream);

/* env.reset() (D:bin3D.py:61-67, C:bin3D.py:69-75) for chosen envs of the batch: start new episodes in some envs and leave the others
 * as they are.  For gym semantics on a whole batch (no_auto_reset = 1: the caller sees the terminal observation, then resets the
 * finished envs), episode control under auto-reset (time limits, curricula, dropping an episode), and device-resident loops, where a
 * captured graph resets on the step's own done bytes (policy -> pct_step -> pct_reset_envs(d_mask = d_done)).
 * Exactly one of d_env / d_mask is non-NULL:
 *   d_env : n env indices.  They must be distinct (caller's contract, as for pct_restore); an index outside [0, n_envs) is skipped.
 *   d_mask: n_envs bytes, n == n_envs; env e resets iff d_mask[e] != 0.  The d_done buffer of the preceding pct_step can be passed as is.
 * A selected env gets exactly what pct_step's auto-reset does to a finished env: counters, sticky flags, the EMS list, boxes and loads
 * are cleared; the draw position is kept (under pct_set_trajectory_length it jumps to the start of the next trajectory,
 * LoadBoxCreator.reset) and a fresh item is drawn.  The current item is discarded, as RandomBoxCreator.reset() discards its list,
 * including an item set by pct_set_items.  An env's items depend on its global id only, so sharding does not change them.  Resets in
 * mid-episode are allowed, with or without no_auto_reset.
 *   d_obs : n_envs x obs_len, every env's observation rows, under the layout and delta-row buffer contract of pct_step
 *   d_info: n_envs pct_step_info records (may be NULL), as pct_set_items writes them: counter, sticky flags, n_leaf, n_cand, n_ems;
 *           ratio / ep_reward / ep_len 0.  (The terminal records are the ones the preceding pct_step wrote.)
 * Enqueue only: no host synchronisation, no allocation (CUDA-graph capturable).  n == 0 (d_env): no-op.  Errors: PCT_ERR_STATE before
 * pct_reset; PCT_ERR_INVALID when both or neither of d_env / d_mask are given, for n < 0, and for a mask with n != n_envs.
 * Whole-batch re-expansion, as for pct_set_items: EVERY env of the handle is re-expanded and gets its rows written to d_obs; envs not
 * selected come out bit-identical.  So the call costs about one pct_step minus its apply kernel however few envs it resets, an
 * all-zero mask included (less when many envs reset: empty bins expand fast).  A caller of the gym loop who keeps the terminal
 * observations must copy them out of d_obs first (the reset overwrites the rows of the reset envs); passing the reset another buffer
 * than the step's forces full row writes. */
int pct_reset_envs(pct_handle h, const int32_t *d_env, int32_t n, const uint8_t *d_mask, void *d_obs, pct_step_info *d_info, void *stream);

/* Snapshot / restore of env states on the device: branch an env (lookahead, beam search, Monte Carlo rollouts), copy it into other
 * slots, move it to another handle or GPU, or checkpoint a batch mid-episode.  Like pct_step, both calls only enqueue kernels on
 * `stream`: no host synchronisation, no allocation (CUDA-graph capturable).
 *
 * A record holds exactly the state that carries over from one step to the next (what a step reads before it writes it: the placed
 * boxes, EMS list, load edges and support polygons, the leaf rows of the last observation, the next item and its draw position, the
 * episode counters and sticky flags, the alias-mode load objects and the LSAH footprint of pct_heuristic_actions*) and nothing
 * transient.  It holds no pointers and no slot-dependent data, so it restores into any slot of any handle with the same
 * configuration, on any device: moving or saving records is a plain byte copy.  Only the live parts of a record are written / read;
 * the record size is fixed per domain so that records can be indexed.  A record starts with a 16-byte header: a layout version and
 * a fingerprint of domain, setting, container, holder sizes, lnes and alias mode.
 *
 * Item source after a restore: the env keeps the record's draw position, but later items come from the slot it now occupies (its
 * own counter-based key in PCT_ITEMS_RANDOM mode, its own stream row, with the trajectory length, in PCT_ITEMS_STREAM mode).  So
 * children of one record restored into different slots sample different futures; a restore into the same slot, or into a slot
 * with the same stream row and global env id, replays exactly the same future. */
/* bytes of one record in a snapshot buffer of this handle (fixed per domain) */
int64_t pct_snapshot_bytes(pct_handle h);
/* gather: record i of d_buf (16-byte aligned, n x pct_snapshot_bytes) <- state of env d_env[i] (d_env NULL: envs 0..n-1).
 * An index outside [0, n_envs) writes a header that no restore accepts. */
int pct_snapshot(pct_handle h, const int32_t *d_env, int32_t n, void *d_buf, void *stream);
/* scatter: env d_env[i] <- record d_rec[i] of d_buf (d_env NULL: env i; d_rec NULL: record i; one record may feed many envs = fan-out).
 *   Destinations within one call must be distinct (caller's contract).  Env indices outside [0, n_envs) and negative record indices
 *   are skipped; record indices must address records inside d_buf.  A record whose header does not match this handle is not applied:
 *   the env stays as it was and gets the sticky PCT_FLAG_BAD_SNAPSHOT, which its next step reports.
 *   d_obs non-NULL: writes the COMPLETE observation rows of every restored env into d_obs (row layout of pct_step, row = env index).
 *   Delta rows: a restored env's next pct_step rewrites all of its rows in whatever buffer it receives, so restoring with d_obs NULL
 *   keeps the observation-buffer contract of pct_step. */
int pct_restore(pct_handle h, const int32_t *d_env, const int32_t *d_rec, int32_t n, const void *d_buf, void *d_obs, void *stream);

/* introspection */
int pct_get_state(pct_handle h, int32_t env, pct_state_dump *out);
/* Same contract as pct_get_state (synchronises the device, copies the env's records to the host, decodes there; no kernel), both
 * domains, both alias modes; setting 2 keeps no graph and yields the empty one.  The stored lists are walked defensively: a cycle, an
 * index beyond n_edge / n_box or an edge filed in two lists returns PCT_ERR_STATE with the finding in pct_last_error. */
int pct_get_support_graph(pct_handle h, int32_t env, pct_support_graph *out);
int32_t pct_obs_len(pct_handle h);       /* (NB + NL + 1) * 9 */
int32_t pct_num_envs(pct_handle h);
int64_t pct_state_bytes_per_env(pct_handle h); /* HBM bytes of library-owned state per env (roofline accounting) */
int64_t pct_kernel_launches(pct_handle h);     /* kernels launched by this handle so far */
/* Per-kernel device timing for roofline accounting: while enabled, every pct_step records CUDA events around its three
 * kernels on the launching stream; pct_profile_read synchronises and returns the summed milliseconds of
 * {apply, candidates, feas_emit} and the number of steps recorded since pct_profile_enable(h, 1). */
int pct_profile_enable(pct_handle h, int32_t on);
int pct_profile_read(pct_handle h, double ms_out[3], int32_t *n_steps);
const char *pct_version(void);

#ifdef __cplusplus
}
#endif
#endif
