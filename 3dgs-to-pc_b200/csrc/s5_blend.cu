// s5_blend.cu — S5: per-leaf front-to-back blend with per-Gaussian max-contribution tracking; S6: accumulate; image.
//
// Reference semantics restated (not copied), renderer_type=python, gauss_render.py:337-402:
//   every Gaussian of a leaf's depth-ordered list contributes to EVERY pixel of the leaf (no 1/255 cut, no early
//   termination, no per-pixel radius test):
//     weight = exp(-0.5 (dx^2 c00 + dy^2 c11 + dx dy c01 + dx dy c10)),  alpha = min(0.99, weight * opacity),
//     contribution = T * alpha,  T <- T (1 - alpha),  pixel = sum contribution * colour + (1 - sum contribution) * bg
//   per Gaussian: the largest contribution over the leaf's pixels and the pixel where it occurs; where that beats the
//   Gaussian's running maximum (strict >, over leaves in BFS order and cameras in call order) the maximum and the
//   blended colour of that pixel are stored (:371-395).
// Role of renderCUDA (forward.cu:303-497) in the reference's CUDA back-end; none of its structure is kept.
//
// Kernel shape: persistent CTAs of 128 threads pull (leaf, slab) items, heaviest leaf first; a CTA owns up to 128 quads
// (4 consecutive pixels of one row) of a leaf and walks the leaf's depth-ordered id list in chunks of 128 Gaussians
// through a 3-deep software pipeline:
//   stage A  the id chunk c+2 is brought into shared memory by ONE TMA bulk copy (cp.async.bulk + mbarrier
//            complete_tx; the lists are 16-byte aligned by the tree kernel)                  — "TMA staging of tile lists"
//   stage B  the 48-byte projection records of chunk c+1 are gathered by cp.async (LDGSTS, 16-byte copies addressed by
//            the staged ids) straight into shared memory, no register round trip
//   stage C  chunk c is blended
// so the dependent id -> record latency of the next chunks hides under the arithmetic of the current one.  Per thread
// and Gaussian the row-dependent terms are formed once; the per-pixel arithmetic is 8 FP32 ops (FADD / FFMA / FMUL, each
// rounded on its own, never contracted) + 1 EX2 + 1 FMNMX per pixel.
// The per-Gaussian maximum is a redux.sync (u32 max of the non-negative float bits) per warp, merged across warps in
// shared memory and published with ONE 64-bit atomicMax per (CTA, Gaussian): key = (contribution bits << 32) |
// ~(leaf-pixel index), so ties go to the earliest leaf / lowest pixel, deterministically.
// Short-cuts: (i) a warp stops once ALL its pixels have T below t_stop (checked every 32 Gaussians): every contribution
// it skips is < t_stop and so is their sum per pixel; t_stop = FLT_MIN in strict-parity runs; (ii) the arg-max
// bookkeeping of a Gaussian is skipped by a warp when none of its contributions exceeds the maximum the Gaussian already
// holds from earlier cameras (the update rule is a strict >, so such contributions can never be recorded); (iii) the
// footprint cull below.
//
// Footprint cull (only when t_stop > FLT_MIN and g2pc_blend_set_cull is on, the default; the strict-parity setting
// t_stop = FLT_MIN runs the kernel instantiated without it).  Every Gaussian of a list reaches every pixel of the leaf,
// but a splat that touches one corner of a leaf is negligible over most of the warps' pixel rectangles.  Per leaf
//     eps = min(2^-26, t_stop / cnt)                                       (cnt: the leaf's list length)
// and at the start of each 32-entry sub-step lane l tests entry j0 + l against the warp's rectangle R (the bounding box
// of its active pixels).  With the record's conic pre-scaled by K = -log2(e)/2, (a, b, c) = (q0.z, q0.w, q1.x), and
// L = log2(opacity) (q1.y), the kernel's exponent is e = L - q(d), q(d) = -(a dx^2 + b dx dy + c dy^2), d = pixel -
// mean, and alpha <= exp2(e).  So alpha < eps on all of R when  min_R q > kappa = L - log2(eps).  For a < 0, c < 0 the
// restriction of q to a line of constant x or y is a convex parabola, and q has no critical point but d = 0, so when
// the mean lies outside R the minimum over R is the least of the four edge minima, each found by clamping the
// parabola's vertex to the edge: the test is exact (not a bounding-box test) and needs no det > 0.  The lane votes
// "skip" only when all of: a < 0, c < 0, 4ac > b^2, the mean is outside R (closed), every term is finite, and
//     min_R q > kappa + 2^-16 S + 2^-12,    S = |L| + |a| Dx^2 + |b| Dx Dy + |c| Dy^2,
// Dx, Dy the largest |dx|, |dy| over R.  The margin: each product of the kernel's e (dx, dy, dy^2, b dy, the two FMAs)
// is rounded at most 5 times, so |e_f32 - e| <= 5 u S (u = 2^-24); the test's own f32 edge minima and S are off by a
// few u S more (the clamped vertex is off by a rounding, which raises q by a second-order amount); together below
// 16 u S = 2^-20 S, taken with 16x headroom.  The absolute 2^-12 covers ex2.approx (relative error < 2^-21, i.e.
// < 2^-20 in log2 units) and the rounding of log2(eps) and kappa (|log2 eps| < 64: a few ulp of 64 = 2^-17).  NaN or
// infinite terms make S or kappa + margin non-finite, and every comparison then keeps the entry.  The warp walks the
// kept entries of the ballot in ascending order, so depth order is unchanged; `iters` counts only those.  Two
// properties follow:
//   * T is bit-identical: a skipped alpha is < 2^-26, so c = T alpha < half an ulp of T and T - c rounds to T.  Every
//     kept contribution is computed bit for bit as without the cull, and so are the per-Gaussian maxima and arg-max
//     pixels of every Gaussian whose maximum is >= 2^-26 (>= eps of every leaf).
//   * bounded colour change: the skipped contributions of a pixel sum to < cnt eps <= t_stop, the same bound as the
//     transmittance stop, so default vs strict still moves a colour by < 2 t_stop x max |colour|.
#include "colour_common.cuh"

namespace {

constexpr int BT = 128;
constexpr int CH = 128;
constexpr int SUB = 32;   // Gaussians between two transmittance checks
constexpr unsigned FULLM = 0xffffffffu;

struct BlendParams {
    const g2pc_leaf_t* leaves;
    const int32_t* leaf_order;
    const int32_t* header;
    const uint32_t* fail;
    int32_t frame;
    const uint32_t* inst_gid;
    const float4* proj;
    unsigned long long* cam_best;
    const float* max_contrib;  // running per-Gaussian maxima of the earlier cameras (threshold for the bookkeeping)
    float* leaf_colour;
    uint32_t* owner;
    int32_t W, H;
    float bg;
    float t_stop;
    int32_t* work_counter;  // cleared by the tree kernel: dynamic (leaf, slab) work distribution
    int32_t slabs;
    int32_t compact;        // 1: compact warp footprints (blocks), 0: row strips
    unsigned long long* stats;
};

// per-lane FP32 on a pixel pair with a scalar operand; the _rn intrinsics keep every op rounded on its own (no FMA
// contraction), which fixes the results bit for bit
__device__ __forceinline__ float2 add2(float2 a, float b) { return make_float2(__fadd_rn(a.x, b), __fadd_rn(a.y, b)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b, c.x), __fmaf_rn(a.y, b, c.y));
}
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float c) {
    return make_float2(__fmaf_rn(a.x, b.x, c), __fmaf_rn(a.y, b.y, c));
}

__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}

// q(d) = -(a dx^2 + b dx dy + c dy^2)
__device__ __forceinline__ float cull_q(float a, float b, float c, float dx, float dy) {
    return -fmaf(dx, fmaf(a, dx, b * dy), c * dy * dy);
}

// footprint cull (header comment): true when alpha < 2^log2eps at every point of the rectangle [x0, x1] x [y0, y1]
__device__ __forceinline__ bool cull_negligible(float4 q0, float4 q1, float x0, float x1, float y0, float y1,
                                                float log2eps) {
    const float a = q0.z, b = q0.w, c = q1.x, L = q1.y;
    const float dx0 = x0 - q0.x, dx1 = x1 - q0.x, dy0 = y0 - q0.y, dy1 = y1 - q0.y;
    const bool inside = dx0 <= 0.0f && dx1 >= 0.0f && dy0 <= 0.0f && dy1 >= 0.0f;
    const float Dx = fmaxf(fabsf(dx0), fabsf(dx1)), Dy = fmaxf(fabsf(dy0), fabsf(dy1));
    const float S = fabsf(L) + fabsf(a) * Dx * Dx + fabsf(b) * Dx * Dy + fabsf(c) * Dy * Dy;
    // edge minima: the parabola along x = const has its vertex at dy = -b dx / (2c), along y = const at dx = -b dy / (2a)
    const float ry = -0.5f * b / c, rx = -0.5f * b / a;
    const float qmin = fminf(fminf(cull_q(a, b, c, dx0, fminf(fmaxf(ry * dx0, dy0), dy1)),
                                   cull_q(a, b, c, dx1, fminf(fmaxf(ry * dx1, dy0), dy1))),
                             fminf(cull_q(a, b, c, fminf(fmaxf(rx * dy0, dx0), dx1), dy0),
                                   cull_q(a, b, c, fminf(fmaxf(rx * dy1, dx0), dx1), dy1)));
    const float kappa = L - log2eps;
    // a finite S bounds every term; finite vertex slopes keep the clamps from meeting inf x 0
    return S + fabsf(rx) + fabsf(ry) < INFINITY && a < 0.0f && c < 0.0f && 4.0f * a * c > b * b && !inside &&
           qmin > kappa + fmaf(S, 0x1p-16f, 0x1p-12f);
}

template <bool CULL>
__global__ void __launch_bounds__(BT, 8) blend_kernel(const BlendParams p) {
    __shared__ __align__(16) float4 s_q0[2][CH];
    __shared__ __align__(16) float4 s_q1[2][CH];
    __shared__ __align__(8) float2 s_b[2][CH];           // (blue, threshold)
    __shared__ __align__(16) uint32_t s_gid[3][CH];      // id chunks, filled by the TMA engine
    __shared__ unsigned long long s_best[BT / 32][CH];
    __shared__ __align__(8) unsigned long long s_bar[3];
    __shared__ int s_item;

    if (g2pc_frame_skipped(p.fail, p.frame)) return;
    const int num_items = p.header[G2PC_HDR_NUM_LEAVES] * p.slabs;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) id_ring_init(s_bar);
    for (int w = 0; w < BT / 32; ++w) s_best[w][tid] = 0ull;
    uint32_t phase_bits = 0;  // parity of the next completion of each id barrier (bit s)
    const float t_stop = p.t_stop;
    unsigned long long iters = 0;
    __syncthreads();

    // persistent CTAs: work items (leaf, slab) are handed out heaviest-leaf-first from a global counter, so the tail of
    // the launch is at most one item long
  for (;;) {
    const int item = next_work_item(p.work_counter, &s_item);
    if (item >= num_items) break;
    const g2pc_leaf_t lf = p.leaves[p.leaf_order[item / p.slabs]];
    const int qpr = (lf.w + 3) >> 2;
    bool active;
    int row, x0;
    if (p.compact) {
        // compact warp footprints: a warp owns a block of tw quad columns x th rows (<= 32 quads, e.g. 20 x 6 pixels of a
        // 40 x 23 leaf) instead of a strip of full rows — the pixels of a block reach the transmittance stop together
        const int ncb = (qpr + 4) / 5;                 // blocks across
        const int tw = (qpr + ncb - 1) / ncb;          // <= 5 quad columns per block
        const int th = 32 / tw;                        // rows per block
        const int nrb = (lf.h + th - 1) / th;
        const int wblock = (item % p.slabs) * (BT / 32) + warp;   // block of this warp
        if ((item % p.slabs) * (BT / 32) >= ncb * nrb) continue;  // uniform: no block left for this slab
        const int bx = wblock % ncb, by = wblock / ncb;
        const int lr = lane / tw, lc = lane - lr * tw;
        row = by * th + lr;
        const int qc = bx * tw + lc;
        active = wblock < ncb * nrb && lr < th && row < lf.h && qc < qpr;
        x0 = qc * 4;
        if (!active) { row = 0; x0 = 0; }
    } else {
        const int nquads = qpr * lf.h;
        const int quad0 = (item % p.slabs) * BT;
        if (quad0 >= nquads) continue;
        const int quad = quad0 + tid;
        active = quad < nquads;
        row = active ? quad / qpr : 0;
        x0 = active ? (quad - row * qpr) * 4 : 0;
    }

    // four pixels per thread, held as two pairs; the per-Gaussian scalars are shared by all four
    float2 T01, T23, px01, px23;
    float2 Cr01 = make_float2(0.f, 0.f), Cr23 = Cr01, Cg01 = Cr01, Cg23 = Cr01, Cb01 = Cr01, Cb23 = Cr01;
    {
        float Tv[4], pxv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const bool valid = active && (x0 + i < lf.w);
            Tv[i] = valid ? 1.0f : 0.0f;  // T = 0 makes every contribution of a padding pixel exactly 0
            pxv[i] = (float)(lf.c0 + x0 + i);
        }
        T01 = make_float2(Tv[0], Tv[1]); T23 = make_float2(Tv[2], Tv[3]);
        px01 = make_float2(pxv[0], pxv[1]); px23 = make_float2(pxv[2], pxv[3]);
    }
    const float py = (float)(lf.r0 + row);
    const int pix_row = row * lf.w + x0;

    const int cnt = lf.inst_count;
    // footprint cull: the warp's rectangle (bounding box of its active pixels; a warp without one has T = 0 everywhere,
    // so whatever it skips changes nothing) and log2 eps = min(-26, log2(t_stop / cnt))
    float rx0 = 0.f, rx1 = 0.f, ry0 = 0.f, ry1 = 0.f, log2eps = 0.f;
    if constexpr (CULL) {
        rx0 = (float)(lf.c0 + (int)__reduce_min_sync(FULLM, active ? (unsigned)x0 : 1u << 30));
        rx1 = (float)(lf.c0 + (int)__reduce_max_sync(FULLM, active ? (unsigned)min(x0 + 3, lf.w - 1) : 0u));
        ry0 = (float)(lf.r0 + (int)__reduce_min_sync(FULLM, active ? (unsigned)row : 1u << 30));
        ry1 = (float)(lf.r0 + (int)__reduce_max_sync(FULLM, active ? (unsigned)row : 0u));
        log2eps = fminf(-26.0f, log2f(t_stop) - log2f((float)cnt));
    }
    const int nchunks = (cnt + CH - 1) / CH;
    const uint32_t* list = p.inst_gid + (int64_t)lf.inst_begin;  // 16-byte aligned (tree kernel)

    // ---- pipeline helpers ------------------------------------------------------------------------------------------
    auto issue_records = [&](int c) {
        const int nl = min(CH, cnt - c * CH);
        if (tid < nl) {
            const uint32_t gid = s_gid[c % 3][tid];
            const float4* rec = p.proj + 3 * (int64_t)gid;
            cp_async16(&s_q0[c & 1][tid], rec);
            cp_async16(&s_q1[c & 1][tid], rec + 1);
            cp_async4(&s_b[c & 1][tid].x, rec + 2);
            cp_async4(&s_b[c & 1][tid].y, p.max_contrib + gid);
        }
        cp_async_commit();
    };

    bool warp_done = false;
    if (nchunks > 0) {
        if (tid == 0) {
            id_ring_issue(s_gid, s_bar, list, cnt, 0);
            if (nchunks > 1) id_ring_issue(s_gid, s_bar, list, cnt, 1);
        }
        id_ring_wait(s_bar, phase_bits, 0);
        issue_records(0);
    }
    for (int c = 0; c < nchunks; ++c) {
        const int nload = min(CH, cnt - c * CH);
        const bool more = (c + 1 < nchunks);
        if (more) { id_ring_wait(s_bar, phase_bits, c + 1); issue_records(c + 1); }
        if (more) cp_async_wait<1>(); else cp_async_wait<0>();
        // records of chunk c visible to the CTA; every thread is past the merge of chunk c - 1 (its id buffer is free)
        const bool all_done = __syncthreads_and(warp_done ? 1 : 0);
        if (all_done) {
            if (more) cp_async_wait<0>();  // drain the gather in flight before the buffers are reused by the next item
            break;
        }
        if (tid == 0 && c + 2 < nchunks) id_ring_issue(s_gid, s_bar, list, cnt, c + 2);
        const float4* q0s = s_q0[c & 1];
        const float4* q1s = s_q1[c & 1];
        const float2* bs = s_b[c & 1];
        if (!warp_done) {
            for (int j0 = 0; j0 < nload; j0 += SUB) {
                const int j1 = min(nload, j0 + SUB);
                auto blend_one = [&](const int j) {
                    const float4 q0 = q0s[j];
                    const float4 q1 = q1s[j];
                    const float2 bt = bs[j];
                    const float bl = bt.x;
                    const float dy = py - q0.y;
                    const float Bq = dy * q0.w;
                    const float Cq = fmaf(dy * dy, q1.x, q1.y);  // + log2(opacity): alpha = min(0.99, exp2(e))
                    const float nmx = -q0.x;
                    const float2 dx01 = add2(px01, nmx);
                    const float2 dx23 = add2(px23, nmx);
                    const float2 e01 = fma2(dx01, fma2(dx01, q0.z, make_float2(Bq, Bq)), Cq);
                    const float2 e23 = fma2(dx23, fma2(dx23, q0.z, make_float2(Bq, Bq)), Cq);
                    const float2 a01 = make_float2(fminf(0.99f, ex2_approx(e01.x)), fminf(0.99f, ex2_approx(e01.y)));
                    const float2 a23 = make_float2(fminf(0.99f, ex2_approx(e23.x)), fminf(0.99f, ex2_approx(e23.y)));
                    const float2 c01 = mul2(T01, a01);
                    const float2 c23 = mul2(T23, a23);
                    Cr01 = fma2(c01, q1.z, Cr01);
                    Cr23 = fma2(c23, q1.z, Cr23);
                    Cg01 = fma2(c01, q1.w, Cg01);
                    Cg23 = fma2(c23, q1.w, Cg23);
                    Cb01 = fma2(c01, bl, Cb01);
                    Cb23 = fma2(c23, bl, Cb23);
                    T01 = fma2(c01, -1.0f, T01);  // T - T*alpha (one rounding)
                    T23 = fma2(c23, -1.0f, T23);
                    // arg-max bookkeeping only if some contribution can beat what the Gaussian already holds
                    const float v = fmaxf(fmaxf(c01.x, c01.y), fmaxf(c23.x, c23.y));
                    if (__any_sync(FULLM, v > bt.y)) {
                        // warp max of the (non-negative) contributions, then the lowest pixel index among the lanes holding it
                        const uint32_t vb = __float_as_uint(v);
                        const uint32_t wm = __reduce_max_sync(FULLM, vb);
                        const int i = (c01.x == v) ? 0 : (c01.y == v) ? 1 : (c23.x == v) ? 2 : 3;
                        const uint32_t pk = (vb == wm) ? (0xFFFFFFFFu - (uint32_t)(pix_row + i)) : 0u;
                        const uint32_t wp = __reduce_max_sync(FULLM, pk);
                        if (lane == 0) s_best[warp][j] = ((unsigned long long)wm << 32) | (unsigned long long)wp;
                    }
                };
                if constexpr (CULL) {
                    // lane l votes for entry j0 + l; the kept entries are walked in ascending (depth) order
                    const bool mine = lane < j1 - j0;
                    unsigned keep = __ballot_sync(FULLM, mine && !cull_negligible(q0s[j0 + lane], q1s[j0 + lane],
                                                                                  rx0, rx1, ry0, ry1, log2eps));
                    iters += (unsigned long long)__popc(keep);
                    while (keep) {
                        blend_one(j0 + __ffs(keep) - 1);
                        keep &= keep - 1u;
                    }
                } else {
                    for (int j = j0; j < j1; ++j) blend_one(j);
                    iters += (unsigned long long)(j1 - j0);
                }
                const float tmax = fmaxf(fmaxf(T01.x, T01.y), fmaxf(T23.x, T23.y));
                warp_done = __all_sync(FULLM, tmax < t_stop);
                if (warp_done) break;
            }
        }
        __syncthreads();  // s_best complete; every warp is past its reads of the record buffers of chunk c
        if (tid < nload) {
            unsigned long long best = s_best[0][tid];
            s_best[0][tid] = 0ull;
#pragma unroll
            for (int w = 1; w < BT / 32; ++w) {
                const unsigned long long o = s_best[w][tid];
                s_best[w][tid] = 0ull;
                best = o > best ? o : best;
            }
            if ((best >> 32) != 0ull) {
                // leaf-local pixel -> index into the concatenated leaf-colour buffer (earlier leaf => smaller index)
                const uint32_t pix = 0xFFFFFFFFu - (uint32_t)best;
                const unsigned long long packed = (best & 0xFFFFFFFF00000000ull) |
                                                  (unsigned long long)(0xFFFFFFFFu - (uint32_t)(lf.pix_offset + pix));
                atomicMax(p.cam_best + s_gid[c % 3][tid], packed);
            }
        }
    }
    // final pixel colours: sum + (1 - sum of contributions) * bg; the second factor equals the final T
    if (active) {
        const float T[4] = {T01.x, T01.y, T23.x, T23.y};
        const float Cr[4] = {Cr01.x, Cr01.y, Cr23.x, Cr23.y};
        const float Cg[4] = {Cg01.x, Cg01.y, Cg23.x, Cg23.y};
        const float Cb[4] = {Cb01.x, Cb01.y, Cb23.x, Cb23.y};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (x0 + i < lf.w) {
                const int64_t lp = (int64_t)lf.pix_offset + pix_row + i;
                float* o = p.leaf_colour + 3 * lp;
                o[0] = fmaf(T[i], p.bg, Cr[i]);
                o[1] = fmaf(T[i], p.bg, Cg[i]);
                o[2] = fmaf(T[i], p.bg, Cb[i]);
                // overlapping leaves: the later BFS entry wins the image pixel (gauss_render.py:369)
                atomicMax(p.owner + (int64_t)(lf.r0 + row) * p.W + (lf.c0 + x0 + i), (uint32_t)lp + 1u);
            }
        }
    }
  }  // work-item loop
    if (p.stats && lane == 0 && iters) atomicAdd(p.stats + G2PC_STAT_WARP_GAUSSIANS, iters);
}

// S6: fold one camera's per-Gaussian winners into the running maxima (strict >, earlier camera wins ties) and fetch
// the blended colour of the winning pixel (gauss_render.py:387-395); clears cam_best for the next camera.
__global__ void __launch_bounds__(256) accumulate_kernel(unsigned long long* __restrict__ cam_best,
                                                         const float* __restrict__ leaf_colour, int64_t n,
                                                         float* __restrict__ max_contrib, float* __restrict__ colours,
                                                         int32_t* __restrict__ first_frame, int32_t frame) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    const unsigned long long b = cam_best[g];
    if (b == 0ull) return;
    cam_best[g] = 0ull;
    const float v = __uint_as_float((uint32_t)(b >> 32));
    if (v > max_contrib[g]) {
        max_contrib[g] = v;
        if (first_frame) first_frame[g] = frame;
        const int64_t idx = (int64_t)(0xFFFFFFFFu - (uint32_t)b);
        colours[3 * g] = leaf_colour[3 * idx];
        colours[3 * g + 1] = leaf_colour[3 * idx + 1];
        colours[3 * g + 2] = leaf_colour[3 * idx + 2];
    }
}

// image = leaf colours where a leaf covers the pixel, else background; flipped left-right (gauss_render.py:402)
__global__ void __launch_bounds__(256) compose_kernel(uint32_t* __restrict__ owner, const float* __restrict__ leaf_colour,
                                                      int W, int H, float bg, float* __restrict__ image) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)W * H) return;
    const int y = (int)(i / W), x = (int)(i - (int64_t)y * W);
    const uint32_t o = owner[i];
    owner[i] = 0u;
    float r = bg, g = bg, b = bg;
    if (o) { const float* c = leaf_colour + 3 * (int64_t)(o - 1u); r = c[0]; g = c[1]; b = c[2]; }
    float* out = image + 3 * ((int64_t)y * W + (W - 1 - x));
    out[0] = r; out[1] = g; out[2] = b;
}

}  // namespace

static int g_blend_compact = 1;
/* experiment switch (bench / tests): 1 = compact warp footprints (default), 0 = row strips */
extern "C" void g2pc_blend_set_compact(int on) { g_blend_compact = on ? 1 : 0; }

static int g_blend_cull = 1;
/* experiment switch (bench / tests): 1 = footprint cull when t_stop > FLT_MIN (default), 0 = never */
extern "C" void g2pc_blend_set_cull(int on) { g_blend_cull = on ? 1 : 0; }

extern "C" int g2pc_blend(const g2pc_leaf_t* leaves, const int32_t* leaf_order, const int32_t* header,
                          const uint32_t* fail, int32_t frame, int32_t max_leaf_width, int32_t max_leaf_height,
                          const uint32_t* inst_gid, const void* proj,
                          uint64_t* cam_best, const float* max_contrib, float* leaf_colour, uint32_t* owner,
                          int32_t width, int32_t height, float background, float t_stop, int32_t* work_counters,
                          uint64_t* stats, void* stream) {
    G2PC_CHECK_ARG(leaves && leaf_order && header && fail && inst_gid && proj && cam_best && max_contrib && leaf_colour &&
                       owner && work_counters, "null pointer");
    G2PC_CHECK_ARG(max_leaf_width >= 1 && max_leaf_height >= 1, "max_leaf_width / max_leaf_height < 1");
    G2PC_CHECK_ARG(t_stop >= 0.0f && t_stop < 1.0f, "t_stop must be in [0, 1)");
    G2PC_CHECK_ARG(((uintptr_t)inst_gid & 15) == 0, "inst_gid must be 16-byte aligned (TMA bulk copies)");
    BlendParams p;
    p.leaves = leaves; p.leaf_order = leaf_order; p.header = header; p.fail = fail; p.frame = frame;
    p.inst_gid = inst_gid;
    p.proj = (const float4*)proj;
    p.cam_best = (unsigned long long*)cam_best; p.max_contrib = max_contrib; p.leaf_colour = leaf_colour;
    p.owner = owner;
    p.W = width; p.H = height; p.bg = background;
    p.t_stop = t_stop > 1.17549435e-38f ? t_stop : 1.17549435e-38f;
    p.compact = g_blend_compact;
    // slabs: work items (CTA-sized parts) per leaf.  Row strips: ceil(quads / 128), quads = ceil(max_w / 4) * max_h.
    // Blocks: 4 per item.  A leaf within max_w x max_h has at most ceil(ceil(max_w / 4) / 5) blocks across (the count
    // grows with the width) and at most ceil(max_h / 6) down (a block has >= 6 rows).  ceil(quads / 100) + 1 items are
    // enough for leaves up to 160 px wide and are kept there (C3: 10 items for 60 x 60 leaves); wider, shorter leaves
    // get the count their blocks need.
    const int64_t qpr = (max_leaf_width + 3) / 4, quads = qpr * max_leaf_height;
    const int64_t blocks = (qpr + 4) / 5 * (((int64_t)max_leaf_height + 5) / 6);
    const int64_t kept = (quads + 4 * 25 - 1) / (4 * 25) + 1, need = (blocks + 3) / 4;
    const int64_t slabs = p.compact ? (need > kept ? need : kept) : (quads + BT - 1) / BT;
    G2PC_CHECK_ARG(slabs <= 0x7FFFFFFF, "max_leaf_width x max_leaf_height too large");
    p.slabs = (int32_t)slabs;
    p.work_counter = work_counters;
    p.stats = (unsigned long long*)stats;
    if (g_blend_cull && p.t_stop > 1.17549435e-38f)
        blend_kernel<true><<<(unsigned)g2pc_resident_ctas(blend_kernel<true>, BT, 0, 8), BT, 0, (cudaStream_t)stream>>>(p);
    else
        blend_kernel<false><<<(unsigned)g2pc_resident_ctas(blend_kernel<false>, BT, 0, 8), BT, 0, (cudaStream_t)stream>>>(p);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_accumulate(uint64_t* cam_best, const float* leaf_colour, int64_t n, float* max_contrib,
                               float* colours, int32_t* first_frame, int32_t frame, void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(cam_best && leaf_colour && max_contrib && colours, "null pointer");
    accumulate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        (unsigned long long*)cam_best, leaf_colour, n, max_contrib, colours, first_frame, frame);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_compose_image(uint32_t* owner, const float* leaf_colour, int32_t width, int32_t height,
                                  float background, float* image, void* stream) {
    G2PC_CHECK_ARG(width > 0 && height > 0, "bad image size");
    G2PC_CHECK_ARG(owner && leaf_colour && image, "null pointer");
    const int64_t n = (int64_t)width * height;
    compose_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(owner, leaf_colour, width, height,
                                                                                    background, image);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
