// Elementwise / re-indexing kernels around the user's net on small boards (SURVEY.md 8 f-3 and the small-board rewrite):
//
//   hrl_board_expand / hrl_board_fold   conv weight (Cout,Cin,kh,kw) <-> the dense matrix (Cout*HW, Cin*HW) of a stride-1
//                                       "same" convolution over an H x W board (fastnet.BoardConv2d), and its adjoint
//   hrl_lstm_gates_fwd / _bwd           the gate arithmetic of a convolutional LSTM cell (reference geister.py:49-56):
//                                       (i, f, o, g) = split(conv output); c' = sig(f) c + sig(i) tanh(g); h' = sig(o) tanh(c')
//   hrl_hidden_visible_fwd / _bwd       the hidden state a recurrent net sees at step t (reference train.py:152-158):
//                                       h * observation_mask, summed over players in the turn-alternating layout
//   hrl_hidden_blend_fwd / _bwd         the hidden state kept after step t (train.py:173): h (1 - m) + h_new m
//
// All are single-pass, coalesced, fp32, one launch each (the eager PyTorch forms are 6-15 launches with temporaries;
// a Geister learner step runs them ~3,000 times, which is what made that step launch-bound).
#include <cuda_bf16.h>
#include <math.h>

#include <cstring>

#include "common.cuh"

namespace hrl {

// ---- dense <-> conv weight ----------------------------------------------------------------------------------------
__global__ void board_expand_kernel(const float *__restrict__ w, float *__restrict__ dense, int Cout, int Cin, int kh, int kw, int H,
                                    int W) {
    const int HW = H * W;
    const long long n = (long long)Cout * HW * Cin * HW;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int col = (int)(idx % (Cin * HW)), row = (int)(idx / (Cin * HW));
        const int o = row / HW, q = row - o * HW, i = col / HW, p = col - i * HW;
        const int a = p / W - q / W + kh / 2, b = p % W - q % W + kw / 2;       // tap that makes output cell q read input cell p
        dense[idx] = (a >= 0 && a < kh && b >= 0 && b < kw) ? __ldg(w + ((long long)(o * Cin + i) * kh + a) * kw + b) : 0.f;
    }
}

__host__ __device__ __forceinline__ int hrl_padded_rows_dev(int N) {      // == hrl_gemm_padded_rows
    int n = (N + 15) / 16 * 16;
    if (n > 256) n = (n + 31) / 32 * 32;
    return n;
}

// dense element (row = (o,q), col = (i,p)) of the convolution, straight into packed B-operand images of the wgmma GEMM
// (csrc/gemm_kernel.cu): image[chunk = k / 32][hi | lo][row][slot (k % 32) / 4 ^ (row & 7)][k % 4]
__device__ __forceinline__ void pack_store(float *image, int n_pad, int row, int k, float v) {
    float hi, lo;
    split_tf32(v, hi, lo);
    const long long chunk = k >> 5;
    const int j = (k & 31) >> 2, e = k & 3;
    float *base = image + chunk * (2ll * n_pad * 32) + (long long)row * 32 + (((j ^ (row & 7)) << 2) + e);
    base[0] = hi;
    base[(long long)n_pad * 32] = lo;
}

// the same element in a bf16 image (HrlGemmArgs.bf16): image[chunk][row][64 bytes, slot (k % 32) / 8 ^ ((row >> 1) & 3)][k % 8]
__device__ __forceinline__ void pack_store_bf16(float *image, int n_pad, int row, int k, float v) {
    const long long chunk = k >> 5;
    const int j = (k & 31) >> 3, e = k & 7;
    __nv_bfloat16 *base = reinterpret_cast<__nv_bfloat16 *>(image) + chunk * ((long long)n_pad * 32) + (long long)row * 32;
    base[((j ^ ((row >> 1) & 3)) << 3) + e] = __float2bfloat16_rn(v);
}

__device__ __forceinline__ void pack_store_any(float *image, int n_pad, int row, int k, float v, bool bf16) {
    if (bf16) pack_store_bf16(image, n_pad, row, k, v);
    else pack_store(image, n_pad, row, k, v);
}

__device__ __forceinline__ void board_pack_body(const HrlPackJob &j, int block, int nblocks) {
    const int HW = j.H * j.W, Cin = j.Cin, kh = j.kh, kw = j.kw, W = j.W;
    const int fwd_pad = hrl_padded_rows_dev(j.fwd_rows), bwd_pad = hrl_padded_rows_dev(j.bwd_rows);
    const long long n = (long long)j.Cout * HW * Cin * HW;
    for (long long idx = (long long)block * blockDim.x + threadIdx.x; idx < n; idx += (long long)nblocks * blockDim.x) {
        const int col = (int)(idx % (Cin * HW)), row = (int)(idx / (Cin * HW));
        const int o = row / HW, q = row - o * HW, i = col / HW, p = col - i * HW;
        const int a = p / W - q / W + kh / 2, b = p % W - q % W + kw / 2;
        const float v = (a >= 0 && a < kh && b >= 0 && b < kw) ? __ldg(j.w + ((long long)(o * Cin + i) * kh + a) * kw + b) : 0.f;
        // rows = output features, reduction = input features
        if (j.image_fwd) pack_store_any(j.image_fwd, fwd_pad, j.fwd_row0 + row, col, v, j.bf16);
        // rows = input features, reduction = output features
        if (j.image_bwd) pack_store_any(j.image_bwd, bwd_pad, col, j.bwd_k0 + row, v, j.bf16);
    }
    if (j.bias && j.bias_cells)          // the convolution's bias, one copy per cell (the product's per-column bias)
        for (int idx = block * blockDim.x + threadIdx.x; idx < j.Cout * HW; idx += nblocks * blockDim.x) j.bias_cells[idx] = __ldg(j.bias + idx / HW);
}

struct PackJobs {
    HrlPackJob job[HRL_MAX_BOARD_JOBS];
    int first_block[HRL_MAX_BOARD_JOBS + 1];
    int n;
    // BatchNorm statistics pivots (hrl_board_pack_many_pivot), in the blocks after the jobs' blocks
    const float *rm[HRL_MAX_BOARD_JOBS], *rv[HRL_MAX_BOARD_JOBS];
    float *pivot[HRL_MAX_BOARD_JOBS];
    int layers, C, HW;
};

__global__ void board_pack_kernel(const PackJobs jobs) {
    if ((int)blockIdx.x >= jobs.first_block[jobs.n]) {
        // pivot = the running mean where |running mean| > 32 running std, else 0 (unshifted sums, bit for bit)
        const int per_layer = (jobs.C * jobs.HW + 255) / 256, b = blockIdx.x - jobs.first_block[jobs.n];
        const int l = b / per_layer, i = (b - l * per_layer) * 256 + threadIdx.x;
        if (i < jobs.C * jobs.HW) {
            const float m = jobs.rm[l][i / jobs.HW], v = jobs.rv[l][i / jobs.HW];
            jobs.pivot[l][i] = m * m > 1024.f * v ? m : 0.f;
        }
        return;
    }
    int k = 0;
    while (k + 1 < jobs.n && (int)blockIdx.x >= jobs.first_block[k + 1]) k++;
    board_pack_body(jobs.job[k], blockIdx.x - jobs.first_block[k], jobs.first_block[k + 1] - jobs.first_block[k]);
}

// one CTA per output channel o and group of input channels: the HW rows of the dense gradient of o (HW * Cin*HW floats per K slice),
// in the group's columns only, are summed over the slices with coalesced reads (fixed order -> deterministic) into shared memory,
// then folded onto the group's taps
struct FoldJobs {
    HrlFoldJob job[HRL_MAX_BOARD_JOBS];
    int first_block[HRL_MAX_BOARD_JOBS + 1];
    int groups[HRL_MAX_BOARD_JOBS];                   // CTAs per output channel (groups of input channels)
    int n;
};

__global__ void board_fold_kernel(const FoldJobs jobs) {
    extern __shared__ float slab[];                   // [HW][c_n]: the HW rows of this CTA's own columns, the input channels i_lo..i_hi
    int jk = 0;
    while (jk + 1 < jobs.n && (int)blockIdx.x >= jobs.first_block[jk + 1]) jk++;
    const HrlFoldJob &J = jobs.job[jk];
    const float *__restrict__ ddense = J.ddense;
    float *__restrict__ dw = J.dw;
    const int splits = J.splits, Cin = J.Cin, kh = J.kh, kw = J.kw, H = J.H, W = J.W, n_groups = jobs.groups[jk];
    const long long split_stride = J.split_stride;
    const int local = blockIdx.x - jobs.first_block[jk];
    const int HW = H * W, cols = Cin * HW, n = HW * cols;
    const int o = local / n_groups, gy = local - o * n_groups;
    const int i_per = (Cin + n_groups - 1) / n_groups, i_lo = gy * i_per, i_hi = min(Cin, i_lo + i_per);
    const int c_lo = i_lo * HW, c_n = (i_hi - i_lo) * HW;          // this CTA's column range
    const float *base = ddense + (long long)o * n;
    // a CTA's elements are few (one input channel: HW*HW): several threads share an element, each summing a contiguous run of
    // the K slices with all its loads in flight at once (one memory round trip instead of splits/8), partial sums combined in
    // slice order through shared memory -- deterministic
    const int n_elem = HW * c_n, n_pad = (n_elem + 31) & ~31;
    const int parts = min((int)blockDim.x / n_pad, splits);
    float *partial = slab + n_elem;                   // [parts][n_pad], behind the slab
    if (parts >= 2) {
        const int part = threadIdx.x / n_pad, e0 = threadIdx.x - part * n_pad;
        if (part < parts && e0 < n_elem) {
            const int e = (e0 / c_n) * cols + c_lo + e0 % c_n;
            const int sp_lo = part * splits / parts, sp_hi = (part + 1) * splits / parts;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            int sp = sp_lo;
            for (; sp + 4 <= sp_hi; sp += 4)
#pragma unroll
                for (int u = 0; u < 4; u++) acc[u] += __ldg(base + (long long)(sp + u) * split_stride + e);
            for (; sp < sp_hi; sp++) acc[0] += __ldg(base + (long long)sp * split_stride + e);
            partial[part * n_pad + e0] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
        }
        __syncthreads();
        if ((int)threadIdx.x < n_elem) {
            const int e0 = threadIdx.x;
            float sum = partial[e0];
            for (int q = 1; q < parts; q++) sum += partial[q * n_pad + e0];
            slab[e0] = sum;
        }
    } else {
        for (int e0 = threadIdx.x; e0 < n_elem; e0 += blockDim.x) {
            const int e = (e0 / c_n) * cols + c_lo + e0 % c_n;
            float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            int sp = 0;
            for (; sp + 8 <= splits; sp += 8) {           // eight independent loads in flight per thread (latency-bound otherwise)
#pragma unroll
                for (int u = 0; u < 8; u++) acc[u] += __ldg(base + (long long)(sp + u) * split_stride + e);
            }
            for (; sp < splits; sp++) acc[0] += __ldg(base + (long long)sp * split_stride + e);
            slab[e0] = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
        }
    }
    __syncthreads();
    const int taps = kh * kw;
    for (int t = threadIdx.x; t < (i_hi - i_lo) * taps; t += blockDim.x) {
        const int i = i_lo + t / taps, a = (t % taps) / kw, b = t % kw;
        float s = 0.f;
        for (int qy = 0; qy < H; qy++) {
            const int py = qy + a - kh / 2;
            if (py < 0 || py >= H) continue;
            for (int qx = 0; qx < W; qx++) {
                const int px = qx + b - kw / 2;
                if (px < 0 || px >= W) continue;
                s += slab[(qy * W + qx) * c_n + (i - i_lo) * HW + py * W + px];
            }
        }
        float *d = dw + ((long long)(o * Cin + i) * kh + a) * kw + b;
        *d = J.accumulate ? *d + s : s;
    }
}

// ---- ConvLSTM gates ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

// gates (N, 4C, S) in the order i, f, o, g; c_prev, h_out, c_out (N, C, S)
__global__ void lstm_gates_fwd_kernel(const float *__restrict__ gates, const float *__restrict__ c_prev, float *__restrict__ h_out,
                                      float *__restrict__ c_out, long long N, int CS) {
    const long long n = N * CS;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const long long b = idx / CS;
        const int r = (int)(idx - b * CS);
        const float *g = gates + b * 4 * CS + r;
        const float i = sigmoid_f(__ldg(g)), f = sigmoid_f(__ldg(g + CS)), o = sigmoid_f(__ldg(g + 2 * CS)), gg = tanhf(__ldg(g + 3 * CS));
        const float c = f * __ldg(c_prev + idx) + i * gg;
        c_out[idx] = c;
        h_out[idx] = o * tanhf(c);
    }
}

// dh, dc_out may be NULL (= 0); writes dgates (N, 4C, S) and dc_prev (N, C, S)
__global__ void lstm_gates_bwd_kernel(const float *__restrict__ gates, const float *__restrict__ c_prev, const float *__restrict__ dh,
                                      const float *__restrict__ dc_out, float *__restrict__ dgates, float *__restrict__ dc_prev,
                                      long long N, int CS) {
    const long long n = N * CS;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const long long b = idx / CS;
        const int r = (int)(idx - b * CS);
        const float *g = gates + b * 4 * CS + r;
        const float i = sigmoid_f(__ldg(g)), f = sigmoid_f(__ldg(g + CS)), o = sigmoid_f(__ldg(g + 2 * CS)), gg = tanhf(__ldg(g + 3 * CS));
        const float cp = __ldg(c_prev + idx);
        const float tc = tanhf(f * cp + i * gg);
        const float gh = dh ? __ldg(dh + idx) : 0.f;
        const float dc = (dc_out ? __ldg(dc_out + idx) : 0.f) + gh * o * (1.f - tc * tc);
        float *dg = dgates + b * 4 * CS + r;
        dg[0] = dc * gg * i * (1.f - i);
        dg[CS] = dc * cp * f * (1.f - f);
        dg[2 * CS] = gh * tc * o * (1.f - o);
        dg[3 * CS] = dc * i * (1.f - gg * gg);
        dc_prev[idx] = dc * f;
    }
}

// ---- hidden state masking (B, P, R) with the step's observation mask om[b*om_stride + p] -------------------------
// sum_players = 1: out (B, R) = sum_p h[b,p,:] om[b,p]   (turn-alternating batches: only the turn player observes)
// sum_players = 0: out (B, P, R) = h om
__global__ void hidden_visible_fwd_kernel(const float *__restrict__ h, const float *__restrict__ om, long long om_stride,
                                          float *__restrict__ out, long long B, int P, int R, int sum_players) {
    const long long n = sum_players ? B * R : B * P * R;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        if (sum_players) {
            const long long b = idx / R;
            const int r = (int)(idx - b * R);
            float s = 0.f;
            for (int p = 0; p < P; p++) s += __ldg(h + (b * P + p) * R + r) * __ldg(om + b * om_stride + p);
            out[idx] = s;
        } else {
            const long long bp = idx / R;
            out[idx] = __ldg(h + idx) * __ldg(om + (bp / P) * om_stride + (bp % P));
        }
    }
}

__global__ void hidden_visible_bwd_kernel(const float *__restrict__ dout, const float *__restrict__ om, long long om_stride,
                                          float *__restrict__ dh, long long B, int P, int R, int sum_players) {
    const long long n = B * P * R;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const long long bp = idx / R;
        const int r = (int)(idx - bp * R);
        const long long b = bp / P;
        const float m = __ldg(om + b * om_stride + (bp % P));
        dh[idx] = m * __ldg(dout + (sum_players ? b * R + r : idx));
    }
}

// out (B, P, R) = h (1 - m) + nh m, nh is (B, Pn, R) with Pn == P or Pn == 1 (broadcast over players)
__global__ void hidden_blend_fwd_kernel(const float *__restrict__ h, const float *__restrict__ nh, const float *__restrict__ om,
                                        long long om_stride, float *__restrict__ out, long long B, int P, int Pn, int R) {
    const long long n = B * P * R;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const long long bp = idx / R;
        const int r = (int)(idx - bp * R);
        const long long b = bp / P;
        const float m = __ldg(om + b * om_stride + (bp % P));
        const float v = __ldg(nh + (Pn == 1 ? b * R + r : idx));
        out[idx] = __ldg(h + idx) * (1.f - m) + v * m;
    }
}

// dh (B, P, R) = dout (1 - m); dnh (B, Pn, R) = dout m (summed over players when Pn == 1); dh may be NULL
__global__ void hidden_blend_bwd_kernel(const float *__restrict__ dout, const float *__restrict__ om, long long om_stride,
                                        float *__restrict__ dh, float *__restrict__ dnh, long long B, int P, int Pn, int R) {
    const long long n = (Pn == 1) ? B * R : B * P * R;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        if (Pn == 1) {
            const long long b = idx / R;
            const int r = (int)(idx - b * R);
            float s = 0.f;
            for (int p = 0; p < P; p++) {
                const float m = __ldg(om + b * om_stride + p);
                const float g = __ldg(dout + (b * P + p) * R + r);
                if (dh) dh[(b * P + p) * R + r] = g * (1.f - m);
                s += g * m;
            }
            dnh[idx] = s;
        } else {
            const long long bp = idx / R;
            const float m = __ldg(om + (bp / P) * om_stride + (bp % P));
            const float g = __ldg(dout + idx);
            if (dh) dh[idx] = g * (1.f - m);
            dnh[idx] = g * m;
        }
    }
}

static inline int grid_for(long long n) {
    long long b = (n + 255) / 256;
    const long long cap = (long long)kNumSM * 8;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace hrl

using namespace hrl;

extern "C" int hrl_board_expand(const float *w, float *dense, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw, int32_t H, int32_t W,
                                void *stream) {
    HRL_REQUIRE(w && dense && Cout > 0 && Cin > 0 && kh > 0 && kw > 0 && H > 0 && W > 0 && (kh & 1) && (kw & 1), HRL_ERR_BAD_ARG,
                "hrl_board_expand: NULL pointer or bad shape (odd kernels only)");
    const long long n = (long long)Cout * Cin * H * W * H * W;
    board_expand_kernel<<<grid_for(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(w, dense, Cout, Cin, kh, kw, H, W);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int32_t hrl_gemm_padded_rows(int64_t N) {
    int n = (int)((N + 15) / 16 * 16);
    if (n > 256) n = (n + 31) / 32 * 32;
    return n;
}

extern "C" size_t hrl_board_pack_floats(int64_t rows, int64_t K) {
    return (size_t)((K + 31) / 32) * 2 * (size_t)hrl_gemm_padded_rows(rows) * 32;
}

// ---- convolutions as implicit products (hrl_gemm_fused conv_mode 1 / 2) -----------------------------------------------
__global__ void conv_pack_kernel(const float *__restrict__ w, int Cout, int Cin, int taps, float *__restrict__ image_fwd, int fwd_pad,
                                 float *__restrict__ image_adj, int adj_pad, int bf16) {
    const int cin_p = (Cin + 31) / 32 * 32, cout_p = (Cout + 31) / 32 * 32;
    const long long n = (long long)Cout * Cin * taps;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(idx % taps), ci = (int)((idx / taps) % Cin), co = (int)(idx / ((long long)taps * Cin));
        const float v = __ldg(w + idx);
        if (image_fwd) pack_store_any(image_fwd, fwd_pad, co, t * cin_p + ci, v, bf16);
        if (image_adj) pack_store_any(image_adj, adj_pad, ci, (taps - 1 - t) * cout_p + co, v, bf16);      // flipped kernel, channels swapped
    }
}

__global__ void conv_wgrad_reduce_kernel(const float *__restrict__ partials, int splits, int ncols, float *__restrict__ dw,
                                         float *__restrict__ db, int Cout, int Cin, int taps, int accumulate) {
    const long long n = (long long)Cout * Cin * taps, slice = (long long)Cout * ncols;
    const long long total = n + (db ? Cout : 0);
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const float *src;
        float *dst;
        if (idx < n) {
            const int t = (int)(idx % taps), ci = (int)((idx / taps) % Cin), co = (int)(idx / ((long long)taps * Cin));
            src = partials + (long long)co * ncols + (long long)t * Cin + ci;
            dst = dw + idx;
        } else {                         // the ones row's column: the bias gradient
            const int co = (int)(idx - n);
            src = partials + (long long)co * ncols + (long long)taps * Cin;
            dst = db + co;
        }
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        int sp = 0;
        for (; sp + 4 <= splits; sp += 4)
#pragma unroll
            for (int u = 0; u < 4; u++) acc[u] += __ldg(src + (long long)(sp + u) * slice);
        for (; sp < splits; sp++) acc[0] += __ldg(src + (long long)sp * slice);
        const float sum = (acc[0] + acc[1]) + (acc[2] + acc[3]);
        *dst = accumulate ? *dst + sum : sum;
    }
}

extern "C" int hrl_conv_geometry(int32_t H, int32_t W, int32_t kh, int32_t kw, int32_t wrap, int16_t *table) {
    HRL_REQUIRE(table && H > 0 && W > 0 && kh > 0 && kw > 0 && (kh & 1) && (kw & 1) && H * W <= 256 && kh * kw <= 9 && H * W * kh * kw <= 256 * 9,
                HRL_ERR_BAD_ARG, "hrl_conv_geometry: odd kernels of at most 9 taps over at most 256 cells");
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++)
            for (int a = 0; a < kh; a++)
                for (int b = 0; b < kw; b++) {
                    int yy = y + a - kh / 2, xx = x + b - kw / 2;
                    int v = HRL_CONV_OUTSIDE;
                    if (wrap) { yy = (yy % H + H) % H; xx = (xx % W + W) % W; }
                    if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = (yy * W + xx) - (y * W + x);
                    table[(y * W + x) * kh * kw + a * kw + b] = (int16_t)v;
                }
    return HRL_OK;
}

extern "C" size_t hrl_conv_pack_floats(int32_t rows, int32_t channels, int32_t taps) {
    return hrl_board_pack_floats(rows, (int64_t)taps * ((channels + 31) / 32 * 32));
}

static int conv_pack(const float *w, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw, float *image_fwd, float *image_adj, int bf16,
                     void *stream) {
    HRL_REQUIRE(w && (image_fwd || image_adj) && Cout > 0 && Cin > 0 && kh > 0 && kw > 0 && (!image_fwd || Cout <= 288) && (!image_adj || Cin <= 288),
                HRL_ERR_BAD_ARG, "hrl_conv_pack: NULL pointer, bad shape or more than 288 operand rows");
    const long long n = (long long)Cout * Cin * kh * kw;
    conv_pack_kernel<<<grid_for(n), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(w, Cout, Cin, kh * kw, image_fwd, hrl_padded_rows_dev(Cout),
                                                                                     image_adj, hrl_padded_rows_dev(Cin), bf16);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_conv_pack(const float *w, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw, float *image_fwd, float *image_adj,
                             void *stream) {
    return conv_pack(w, Cout, Cin, kh, kw, image_fwd, image_adj, 0, stream);
}

extern "C" int hrl_conv_pack_bf16(const float *w, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw, float *image_fwd, float *image_adj,
                                  void *stream) {
    return conv_pack(w, Cout, Cin, kh, kw, image_fwd, image_adj, 1, stream);
}

extern "C" int hrl_conv_wgrad_reduce2(const float *partials, int32_t splits, int32_t ncols, float *dw, float *db, int32_t Cout, int32_t Cin,
                                      int32_t taps, int32_t accumulate, void *stream) {
    HRL_REQUIRE(partials && dw && splits >= 1 && Cout > 0 && Cin > 0 && taps > 0 && ncols >= taps * Cin + (db ? 1 : 0), HRL_ERR_BAD_ARG,
                "hrl_conv_wgrad_reduce: NULL pointer or bad shape");
    conv_wgrad_reduce_kernel<<<grid_for((long long)Cout * Cin * taps + Cout), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        partials, splits, ncols, dw, db, Cout, Cin, taps, accumulate);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_conv_wgrad_reduce(const float *partials, int32_t splits, float *dw, int32_t Cout, int32_t Cin, int32_t taps, void *stream) {
    return hrl_conv_wgrad_reduce2(partials, splits, taps * Cin, dw, nullptr, Cout, Cin, taps, 0, stream);
}

extern "C" int hrl_board_pack_many_pivot(const HrlPackJob *jobs, int32_t n_jobs, const float *const *running_mean, const float *const *running_var,
                                         float *const *pivot_col, int32_t layers, int32_t C, int32_t HW, void *stream) {
    HRL_REQUIRE((jobs || n_jobs == 0) && n_jobs >= 0 && n_jobs <= HRL_MAX_BOARD_JOBS && layers >= 0 && layers <= HRL_MAX_BOARD_JOBS &&
                    n_jobs + layers >= 1,
                HRL_ERR_BAD_ARG, "hrl_board_pack_many: 1..%d jobs and 0..%d pivot layers", HRL_MAX_BOARD_JOBS, HRL_MAX_BOARD_JOBS);
    HRL_REQUIRE(layers == 0 || (running_mean && running_var && pivot_col && C > 0 && HW > 0), HRL_ERR_BAD_ARG,
                "hrl_board_pack_many_pivot: NULL pointer or bad shape");
    PackJobs pj;
    pj.n = n_jobs;
    pj.layers = layers; pj.C = C; pj.HW = HW;
    for (int l = 0; l < layers; l++) {
        HRL_REQUIRE(running_mean[l] && running_var[l] && pivot_col[l], HRL_ERR_BAD_ARG, "hrl_board_pack_many_pivot: NULL pointer");
        pj.rm[l] = running_mean[l]; pj.rv[l] = running_var[l]; pj.pivot[l] = pivot_col[l];
    }
    pj.first_block[0] = 0;
    for (int k = 0; k < n_jobs; k++) {
        const HrlPackJob &j = jobs[k];
        HRL_REQUIRE(j.w && (j.image_fwd || j.image_bwd) && j.Cout > 0 && j.Cin > 0 && j.kh > 0 && j.kw > 0 && j.H > 0 && j.W > 0 && (j.kh & 1) &&
                        (j.kw & 1),
                    HRL_ERR_BAD_ARG, "hrl_board_pack: NULL pointer or bad shape (odd kernels only)");
        HRL_REQUIRE((!j.image_fwd || (j.fwd_rows <= 288 && j.fwd_row0 >= 0 && j.fwd_row0 + j.Cout * j.H * j.W <= j.fwd_rows)) &&
                        (!j.image_bwd || (j.bwd_rows <= 288 && j.bwd_rows == j.Cin * j.H * j.W && j.bwd_k0 >= 0)),
                    HRL_ERR_BAD_ARG, "hrl_board_pack: operand rows outside the packed range (<= 288)");
        HRL_REQUIRE((j.bias == nullptr) == (j.bias_cells == nullptr), HRL_ERR_BAD_ARG, "hrl_board_pack: bias and bias_cells go together");
        pj.job[k] = j;
        const long long n = (long long)j.Cout * j.Cin * j.H * j.W * j.H * j.W;
        int blocks = (int)((n + 255) / 256);
        if (blocks > 2 * kNumSM) blocks = 2 * kNumSM;
        pj.first_block[k + 1] = pj.first_block[k] + blocks;
    }
    const int pivot_blocks = layers ? layers * ((C * HW + 255) / 256) : 0;
    board_pack_kernel<<<pj.first_block[n_jobs] + pivot_blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(pj);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_board_pack_many(const HrlPackJob *jobs, int32_t n_jobs, void *stream) {
    HRL_REQUIRE(jobs && n_jobs >= 1, HRL_ERR_BAD_ARG, "hrl_board_pack_many: 1..%d jobs", HRL_MAX_BOARD_JOBS);
    return hrl_board_pack_many_pivot(jobs, n_jobs, nullptr, nullptr, nullptr, 0, 0, 0, stream);
}

extern "C" int hrl_board_pack(const float *w, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw, int32_t H, int32_t W, float *image_fwd,
                              int32_t fwd_rows, int32_t fwd_row0, float *image_bwd, int32_t bwd_rows, int32_t bwd_k0, void *stream) {
    HrlPackJob j;
    memset(&j, 0, sizeof(j));
    j.w = w; j.Cout = Cout; j.Cin = Cin; j.kh = kh; j.kw = kw; j.H = H; j.W = W;
    j.image_fwd = image_fwd; j.fwd_rows = fwd_rows; j.fwd_row0 = fwd_row0;
    j.image_bwd = image_bwd; j.bwd_rows = bwd_rows; j.bwd_k0 = bwd_k0;
    return hrl_board_pack_many(&j, 1, stream);
}

extern "C" int hrl_board_fold_many(const HrlFoldJob *jobs, int32_t n_jobs, void *stream) {
    HRL_REQUIRE(jobs && n_jobs >= 1 && n_jobs <= HRL_MAX_BOARD_JOBS, HRL_ERR_BAD_ARG, "hrl_board_fold_many: 1..%d jobs", HRL_MAX_BOARD_JOBS);
    FoldJobs fj;
    fj.n = n_jobs;
    fj.first_block[0] = 0;
    size_t slab_max = 0;
    for (int k = 0; k < n_jobs; k++) {
        const HrlFoldJob &j = jobs[k];
        HRL_REQUIRE(j.ddense && j.dw && j.splits >= 1 && j.Cout > 0 && j.Cin > 0 && j.kh > 0 && j.kw > 0 && j.H > 0 && j.W > 0 && (j.kh & 1) &&
                        (j.kw & 1),
                    HRL_ERR_BAD_ARG, "hrl_board_fold: NULL pointer or bad shape (odd kernels only)");
        fj.job[k] = j;
        // (output channel, group of input channels) CTAs: at least about two per SM, and few enough elements per CTA (<= 128) that
        // several threads can share the K slices of one element
        int groups = (2 * kNumSM + j.Cout - 1) / j.Cout;
        const int cells2 = j.H * j.W * j.H * j.W, i_max = cells2 >= 128 ? 1 : 128 / cells2;
        if (groups < (j.Cin + i_max - 1) / i_max) groups = (j.Cin + i_max - 1) / i_max;
        if (groups > j.Cin) groups = j.Cin;
        const int i_per = (j.Cin + groups - 1) / groups;      // input channels per CTA, as the kernel splits them
        groups = (j.Cin + i_per - 1) / i_per;                 // the same split, with no CTA left without a channel
        // a CTA's slab holds the rows of its own columns only, + the slice-run partials
        const size_t slab_bytes = ((size_t)j.H * j.W * j.H * j.W * i_per + 512) * sizeof(float);
        HRL_REQUIRE(slab_bytes <= 200 * 1024, HRL_ERR_UNSUPPORTED, "hrl_board_fold: (H*W)^2 x %d channels = %zu floats exceed shared memory",
                    i_per, slab_bytes / sizeof(float));
        if (slab_bytes > slab_max) slab_max = slab_bytes;
        fj.groups[k] = groups;
        fj.first_block[k + 1] = fj.first_block[k] + j.Cout * groups;
    }
    if (slab_max > 48 * 1024)
        HRL_CUDA_CHECK(cudaFuncSetAttribute(board_fold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)slab_max));
    board_fold_kernel<<<fj.first_block[n_jobs], 512, slab_max, reinterpret_cast<cudaStream_t>(stream)>>>(fj);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_board_fold(const float *ddense, int32_t splits, int64_t split_stride, float *dw, int32_t Cout, int32_t Cin, int32_t kh,
                              int32_t kw, int32_t H, int32_t W, void *stream) {
    HrlFoldJob j;
    memset(&j, 0, sizeof(j));
    j.ddense = ddense; j.splits = splits; j.split_stride = split_stride; j.dw = dw;
    j.Cout = Cout; j.Cin = Cin; j.kh = kh; j.kw = kw; j.H = H; j.W = W;
    return hrl_board_fold_many(&j, 1, stream);
}

extern "C" int hrl_lstm_gates_fwd(const float *gates, const float *c_prev, float *h_out, float *c_out, int64_t N, int32_t C, int32_t S,
                                  void *stream) {
    HRL_REQUIRE(gates && c_prev && h_out && c_out && N > 0 && C > 0 && S > 0, HRL_ERR_BAD_ARG, "hrl_lstm_gates_fwd: NULL pointer or bad shape");
    lstm_gates_fwd_kernel<<<grid_for(N * C * S), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(gates, c_prev, h_out, c_out, N, C * S);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_lstm_gates_bwd(const float *gates, const float *c_prev, const float *dh, const float *dc_out, float *dgates,
                                  float *dc_prev, int64_t N, int32_t C, int32_t S, void *stream) {
    HRL_REQUIRE(gates && c_prev && dgates && dc_prev && N > 0 && C > 0 && S > 0, HRL_ERR_BAD_ARG, "hrl_lstm_gates_bwd: NULL pointer or bad shape");
    lstm_gates_bwd_kernel<<<grid_for(N * C * S), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(gates, c_prev, dh, dc_out, dgates, dc_prev,
                                                                                                  N, C * S);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_hidden_visible_fwd(const float *h, const float *om, int64_t om_stride, float *out, int64_t B, int32_t P, int32_t R,
                                      int32_t sum_players, void *stream) {
    HRL_REQUIRE(h && om && out && B > 0 && P > 0 && R > 0, HRL_ERR_BAD_ARG, "hrl_hidden_visible_fwd: NULL pointer or bad shape");
    hidden_visible_fwd_kernel<<<grid_for(sum_players ? B * R : B * P * R), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        h, om, om_stride, out, B, P, R, sum_players);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_hidden_visible_bwd(const float *dout, const float *om, int64_t om_stride, float *dh, int64_t B, int32_t P, int32_t R,
                                      int32_t sum_players, void *stream) {
    HRL_REQUIRE(dout && om && dh && B > 0 && P > 0 && R > 0, HRL_ERR_BAD_ARG, "hrl_hidden_visible_bwd: NULL pointer or bad shape");
    hidden_visible_bwd_kernel<<<grid_for(B * P * R), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(dout, om, om_stride, dh, B, P, R,
                                                                                                      sum_players);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_hidden_blend_fwd(const float *h, const float *nh, const float *om, int64_t om_stride, float *out, int64_t B, int32_t P,
                                    int32_t Pn, int32_t R, void *stream) {
    HRL_REQUIRE(h && nh && om && out && B > 0 && P > 0 && R > 0 && (Pn == 1 || Pn == P), HRL_ERR_BAD_ARG,
                "hrl_hidden_blend_fwd: NULL pointer or bad shape");
    hidden_blend_fwd_kernel<<<grid_for(B * P * R), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(h, nh, om, om_stride, out, B, P, Pn, R);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}

extern "C" int hrl_hidden_blend_bwd(const float *dout, const float *om, int64_t om_stride, float *dh, float *dnh, int64_t B, int32_t P,
                                    int32_t Pn, int32_t R, void *stream) {
    HRL_REQUIRE(dout && om && dnh && B > 0 && P > 0 && R > 0 && (Pn == 1 || Pn == P), HRL_ERR_BAD_ARG,
                "hrl_hidden_blend_bwd: NULL pointer or bad shape");
    hidden_blend_bwd_kernel<<<grid_for(Pn == 1 ? B * R : B * P * R), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(dout, om, om_stride, dh,
                                                                                                                      dnh, B, P, Pn, R);
    HRL_CUDA_CHECK(cudaGetLastError());
    return HRL_OK;
}
