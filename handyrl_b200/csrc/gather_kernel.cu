// K2 -- replay gather/pad: the device form of make_batch (handyrl/train.py:33-124).
//
// Episodes live decoded in a flat "replay store" in HBM (one row per step, see HrlGatherArgs);
// a batch is B window descriptors.  One CTA writes `cells_per_block` consecutive (b,t) cells of
// every batch tensor: live cells copy from the store, cells outside the window get the pad
// constants of train.py:92-106 (prob 1, action_mask 1e32, progress 1, value = outcome after
// the end, everything else 0).  Every batch byte is written exactly once, coalesced along the
// innermost dimension; the store is read once.
//
// hrl_gather_pad_sym is the same kernel with board-symmetry augmentation: window b is written
// through transform sym[b] of a table set (obs_src / act_src / act_dst, see hrl_b200.h).  Live
// observation and action-mask rows are permuted copies, live actions are remapped; every other
// tensor and every pad value is what hrl_gather_pad writes.
#include "common.cuh"

namespace hrl {

struct CellSrc {
    int64_t row;   // store row of this cell's step, or -1 when the cell is padding
    int after;     // padding after the end of the window (value = outcome, train.py:98)
    int step;      // episode step index
};

__device__ __forceinline__ CellSrc locate(const HrlWindow &w, int t, int burn_in) {
    CellSrc c;
    const int len = w.end - w.start;
    const int pad_b = burn_in - (w.train_start - w.start);  // train.py:94
    const int k = t - pad_b;
    c.step = w.start + k;
    c.after = (k >= len);
    c.row = (k >= 0 && k < len) ? (w.first_step + c.step) : -1;
    return c;
}

// copy n floats src -> dst (or fill when src == nullptr) by one warp, 16 bytes per lane when both sides allow it
__device__ __forceinline__ void warp_copy_row(float *__restrict__ dst, const float *__restrict__ src, float fill, int n, int lane) {
    const bool vec = ((n & 3) == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) &&
                     (src == nullptr || (reinterpret_cast<uintptr_t>(src) & 15) == 0);
    if (vec) {
        const int n4 = n >> 2;
        float4 *d4 = reinterpret_cast<float4 *>(dst);
        if (src) {
            const float4 *s4 = reinterpret_cast<const float4 *>(src);
#pragma unroll 4
            for (int i = lane; i < n4; i += 32) __stcs(d4 + i, __ldcs(s4 + i));
        } else {
            const float4 f4 = make_float4(fill, fill, fill, fill);
            for (int i = lane; i < n4; i += 32) __stcs(d4 + i, f4);
        }
    } else {
        if (src) for (int i = lane; i < n; i += 32) dst[i] = src[i];
        else for (int i = lane; i < n; i += 32) dst[i] = fill;
    }
}

// true when tab[e] == e for every e < n (a whole warp votes; stops at the first chunk that differs)
__device__ __forceinline__ bool warp_row_is_identity(const int32_t *__restrict__ tab, int n, int lane) {
    if (((n & 3) == 0) && ((reinterpret_cast<uintptr_t>(tab) & 15) == 0)) {
        const int4 *t4 = reinterpret_cast<const int4 *>(tab);
        for (int i0 = 0; i0 < (n >> 2); i0 += 32) {
            const int i = i0 + lane, e = 4 * i;
            bool ok = true;
            if (i < (n >> 2)) {
                const int4 v = __ldg(t4 + i);
                ok = v.x == e && v.y == e + 1 && v.z == e + 2 && v.w == e + 3;
            }
            if (!__all_sync(0xffffffffu, ok)) return false;
        }
        return true;
    }
    for (int e0 = 0; e0 < n; e0 += 32) {
        const int e = e0 + lane;
        if (!__all_sync(0xffffffffu, e >= n || __ldg(tab + e) == e)) return false;
    }
    return true;
}

// dst[e] = src[tab[e]] for e < n by one warp: writes (and table reads) coalesced along dst, 16 bytes per lane when
// the shapes allow it; the source row is a few hundred bytes to a few KB, so its scattered reads hit L1.  An identity
// row takes warp_copy_row's streaming path instead.
__device__ __forceinline__ void warp_permute_row(float *__restrict__ dst, const float *__restrict__ src,
                                                 const int32_t *__restrict__ tab, int n, int lane) {
    if (warp_row_is_identity(tab, n, lane)) {
        warp_copy_row(dst, src, 0.0f, n, lane);
        return;
    }
    const bool vec = ((n & 3) == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(tab) & 15) == 0);
    if (vec) {
        const int n4 = n >> 2;
        float4 *d4 = reinterpret_cast<float4 *>(dst);
        const int4 *t4 = reinterpret_cast<const int4 *>(tab);
#pragma unroll 2
        for (int i = lane; i < n4; i += 32) {
            const int4 j = __ldg(t4 + i);
            __stcs(d4 + i, make_float4(__ldg(src + j.x), __ldg(src + j.y), __ldg(src + j.z), __ldg(src + j.w)));
        }
    } else {
        for (int i = lane; i < n; i += 32) dst[i] = __ldg(src + __ldg(tab + i));
    }
}

// Tables of hrl_gather_pad_sym (unused when SYM is false).
struct SymTables {
    const int32_t *sym, *obs_src, *act_src, *act_dst;
};

// One warp per (cell, policy row): it locates the source step once and streams the observation and the
// action-mask row (vectorised); lanes then write the handful of per-player scalars of the cell.  SYM: live rows of window b
// go through transform sym[b] (all steps and policy rows of a window alike); the per-cell scalars are untouched.
template <bool SYM>
__global__ void __launch_bounds__(256) gather_pad_kernel(const HrlGatherArgs g, int cells_per_block, const SymTables st) {
    const int T = g.T, P = g.P, Pa = g.Pa, A = g.A, Ps = g.Ps, OE = g.obs_elems;
    const int64_t ncell = (int64_t)g.B * T;
    const int64_t c0 = (int64_t)blockIdx.x * cells_per_block;
    const int nc = (int)min((int64_t)cells_per_block, ncell - c0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    const bool solo = (P == 1 && Ps > 1);

    for (int u = warp; u < nc * Pa; u += nwarp) {
        const int c = u / Pa, q = u - c * Pa;
        const int64_t cell = c0 + c;
        const int b = (int)(cell / T), t = (int)(cell - (int64_t)b * T);
        const HrlWindow w = g.windows[b];
        const CellSrc s = locate(w, t, g.burn_in);
        const bool live = s.row >= 0;
        // policy-side player of row q in this cell (train.py:65-68)
        const int pl = !live ? 0 : (g.turn_alternating ? g.st_turn[s.row] : (solo ? w.player : q));
        const int64_t sp = live ? s.row * Ps + pl : 0;
        const int k = SYM ? st.sym[b] : 0;   // trusted: the caller checked 0 <= sym[b] < K on the host
        if (SYM && live) {
            if (OE > 0) warp_permute_row(g.observation + (cell * Pa + q) * OE, g.st_obs + sp * OE, st.obs_src + (int64_t)k * OE, OE, lane);
            warp_permute_row(g.action_mask + (cell * Pa + q) * A, g.st_amask + sp * A, st.act_src + (int64_t)k * A, A, lane);
        } else {
            if (OE > 0) warp_copy_row(g.observation + (cell * Pa + q) * OE, live ? g.st_obs + sp * OE : nullptr, 0.0f, OE, lane);
            warp_copy_row(g.action_mask + (cell * Pa + q) * A, live ? g.st_amask + sp * A : nullptr, 1e32f, A, lane);
        }
        if (lane == 0) {
            g.selected_prob[cell * Pa + q] = live ? g.st_prob[sp] : 1.0f;
            int32_t a = live ? g.st_action[sp] : 0;
            if (SYM && live && a >= 0 && a < A) a = st.act_dst[(int64_t)k * A + a];
            g.action[cell * Pa + q] = (int64_t)a;
        }
        if (q == 0) {   // the cell's value-side and per-cell scalars, once
            for (int p = lane; p < P; p += 32) {
                const int vp = solo ? w.player : p;
                float val = 0.f, rew = 0.f, ret = 0.f, tm = 0.f, om = 0.f;
                if (live) {
                    const int64_t sv = s.row * Ps + vp;
                    val = g.st_value[sv];
                    rew = g.st_reward[sv];
                    ret = g.st_return[sv];
                    const uint8_t f = g.st_flags[sv];
                    tm = (f & 1) ? 1.0f : 0.0f;
                    om = (f & 2) ? 1.0f : 0.0f;
                } else if (s.after) {
                    val = g.st_outcome[(int64_t)w.outcome_row * Ps + vp];  // np.tile(oc, ...) train.py:98
                }
                const int64_t o = cell * P + p;
                g.value[o] = val;
                g.reward[o] = rew;
                g.ret[o] = ret;
                g.turn_mask[o] = tm;
                g.observation_mask[o] = om;
                if (t == 0) g.outcome[(int64_t)b * P + p] = g.st_outcome[(int64_t)w.outcome_row * Ps + vp];
            }
            if (lane == 0) {
                g.episode_mask[cell] = live ? 1.0f : 0.0f;
                g.progress[cell] = live ? (float)s.step / (float)w.total : 1.0f;  // train.py:89, 106
            }
        }
    }
}

}  // namespace hrl

namespace {

int check_gather_args(const HrlGatherArgs *args, const char *fn) {
    using namespace hrl;
    HRL_REQUIRE(args != nullptr, HRL_ERR_BAD_ARG, "%s: args is NULL", fn);
    const HrlGatherArgs &g = *args;
    HRL_REQUIRE(g.B > 0 && g.T > 0 && g.P > 0 && g.A > 0 && g.Ps > 0 && g.obs_elems >= 0, HRL_ERR_BAD_ARG,
                "%s: non-positive dimension", fn);
    HRL_REQUIRE(g.Pa == 1 || g.Pa == g.P, HRL_ERR_BAD_ARG, "%s: Pa must be 1 or P", fn);
    HRL_REQUIRE(g.P == g.Ps || g.P == 1, HRL_ERR_BAD_ARG, "%s: P must equal Ps, or 1 for solo training", fn);
    HRL_REQUIRE(g.burn_in >= 0 && g.burn_in < g.T, HRL_ERR_BAD_ARG, "%s: burn_in outside [0,T)", fn);
    HRL_REQUIRE(g.windows && g.st_prob && g.st_action && g.st_amask && g.st_value && g.st_reward && g.st_return &&
                    g.st_flags && g.st_outcome && (g.obs_elems == 0 || g.st_obs) && (!g.turn_alternating || g.st_turn),
                HRL_ERR_BAD_ARG, "%s: a replay-store pointer is NULL", fn);
    HRL_REQUIRE(g.selected_prob && g.value && g.action && g.outcome && g.reward && g.ret && g.episode_mask &&
                    g.turn_mask && g.observation_mask && g.action_mask && g.progress && (g.obs_elems == 0 || g.observation),
                HRL_ERR_BAD_ARG, "%s: a batch output pointer is NULL", fn);
    return HRL_OK;
}

template <bool SYM>
int launch_gather(const HrlGatherArgs &g, const hrl::SymTables &st, void *stream) {
    using namespace hrl;
    // 8 warps per CTA, one (cell, policy row) per warp at a time; a CTA takes enough cells for ~16 KB of copies
    const int64_t per_cell = (int64_t)g.Pa * (g.obs_elems + g.A) + 2 * g.Pa + 5 * g.P + 2;
    int cpb = (int)(4096 / per_cell);
    if (cpb < (8 + g.Pa - 1) / g.Pa) cpb = (8 + g.Pa - 1) / g.Pa;
    const int64_t ncell = (int64_t)g.B * g.T;
    // keep at least ~4 CTAs per SM in flight when the batch is small
    while (cpb > 1 && (ncell + cpb - 1) / cpb < 4 * kNumSM) cpb >>= 1;
    const int64_t grid = (ncell + cpb - 1) / cpb;
    gather_pad_kernel<SYM><<<(unsigned)grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(g, cpb, st);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

}  // namespace

extern "C" int hrl_gather_pad(const HrlGatherArgs *args, void *stream) {
    const int rc = check_gather_args(args, "hrl_gather_pad");
    if (rc != HRL_OK) return rc;
    return launch_gather<false>(*args, hrl::SymTables{nullptr, nullptr, nullptr, nullptr}, stream);
}

extern "C" int hrl_gather_pad_sym(const HrlGatherArgs *args, const int32_t *sym, const int32_t *obs_src, const int32_t *act_src,
                                  const int32_t *act_dst, int32_t K, void *stream) {
    using namespace hrl;
    const int rc = check_gather_args(args, "hrl_gather_pad_sym");
    if (rc != HRL_OK) return rc;
    HRL_REQUIRE(K >= 1 && K <= HRL_SYM_MAX_TRANSFORMS, HRL_ERR_BAD_ARG, "hrl_gather_pad_sym: K=%d outside [1,%d]", (int)K,
                HRL_SYM_MAX_TRANSFORMS);
    HRL_REQUIRE(sym && act_src && act_dst && (args->obs_elems == 0 || obs_src), HRL_ERR_BAD_ARG,
                "hrl_gather_pad_sym: a transform table pointer is NULL");
    return launch_gather<true>(*args, SymTables{sym, obs_src, act_src, act_dst}, stream);
}
