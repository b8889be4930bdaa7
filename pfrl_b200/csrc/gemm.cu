// gemm.cu -- K10: the dense layers of the Q-networks on the Hopper tensor cores (wgmma).
//
//   C[M,N] = A[M,K] . B[N,K]^T (+ bias[N]) (relu)          fp32 in, fp32 out
//
// Replaces the cuBLAS SGEMMs behind (reference, all fp32 on the CUDA cores):
//   pfrl/q_functions/dueling_dqn.py:67-129     main_stream / a_stream / v_stream Linear
//   pfrl/nn/noisy_linear.py:53-70              F.linear with the noisy weight
//   pfrl/nn/atari_cnn.py:17-47                 the Linear(3136, 512) head of the Nature nets
// and their two backward products (dX = dY . W, dW = dY^T . X).
//
// Arithmetic: every fp32 operand x is split into two TF32 numbers, x = hi + lo with
// hi = rn_tf32(x), lo = rn_tf32(x - hi), and the product is accumulated as
// lo.hi + hi.lo + hi.hi with `wgmma.mma_async ... .f32.tf32.tf32` (the lo.lo term, <= 2^-22
// relative, is dropped).  That keeps the result within a few fp32 ulps of an exact fp32
// product -- tests/test_gemm_gpu.py measures it against an fp64 product next to cuBLAS' own
// fp32 error -- which is what lets the agents' 1e-5 loss parity stand.
//
// Data movement: no TMA tensor maps.  The split has to touch every element anyway, so all
// sixteen warps read the fp32 tiles through the read-only path, split them in registers and
// store hi and lo straight into the canonical no-swizzle K-major core-matrix layout the tensor
// core reads (8 rows x 16 B per core matrix, K-neighbours padded to 144 B so that every
// quarter warp stores to 8 different bank groups).  Operands whose contraction index is the
// contiguous one ("K-major": X and W in the forward product) are read with 16-byte loads, four
// whole 128-byte rows per warp instruction;
// operands whose contraction index is the ROW index ("MN-major": dY and X in dW = dY^T . X,
// W in dX = dY . W) are read with four 4-byte loads per thread, each warp instruction one
// coalesced 128-byte run along M/N, and the four k values meet in one 16-byte store -- the
// transposition happens in registers, no transposed copy is ever made and the tensor core only
// ever sees K-major tiles (wgmma accepts MN-major operands only for 16-bit types).
// The loads of k block i+1 are in flight while the tensor cores work on block i.
//
// A CTA of four warpgroups computes one 128 x bn output tile (x one K split); bn = 32, 64 or
// 128 by N.  Every warpgroup loads a quarter of each stage and owns a 64 x bn/2 quadrant of the
// tile, held in registers as two accumulators (hi.hi, and lo.hi + hi.lo).  The operand ring has
// 3 stages of (A_hi, A_lo, B_hi, B_lo) = 72 KB; one __syncthreads per k block publishes a stage,
// and each warpgroup keeps at most one wgmma group in flight, so that a stage is rewritten
// only after every warpgroup has finished reading it.  The epilogue adds the two accumulators,
// stages the tile through the idle ring and writes it out in whole rows (dense outputs) or
// coalesced along the rows (NCHW scatter outputs), with bias / relu.
// Small products are split along K so that the grid covers the SMs; the partial tiles go to a
// workspace and `k_gemm_reduce` adds them in a fixed order (deterministic), with the bias /
// relu epilogue.
//
// Convolutions (pfrl/nn/atari_cnn.py:30-44, pfrl/q_functions/dueling_dqn.py:34-40,91-97: the
// 4x4/2 and 3x3/1 layers of the Nature trunk, forward, input gradient, weight gradient) are the
// same product with one more operand mode, "gather": element (row, k) lives at
//   row_off[row] + k_off[k]
// and, when the operand carries coordinates, exists iff 0 <= y[row] + dy[k] < y_limit and
// 0 <= x[row] + dx[k] < x_limit -- im2col, its transpose (col2im as a gather; a strided layer
// is one product per stride phase) and the pixel-major views of the weight gradient, all read
// in place through small int32 tables per operand (ops/conv.py builds them once per layer
// shape).  The output can be scattered the same way (C[m, n] at row_off[m] + n * col_stride:
// NCHW activations and transposed weight gradients), so no im2col buffer and no layout pass
// ever touches HBM.  uint8 sources
// (float(byte) * scale: the x / 255 of the Atari phi) are read directly.
#include "b2rl_internal.cuh"

namespace {

constexpr int BM = 128, BK = 32; // BK floats = 128 bytes of contraction per stage
constexpr int STAGES = 3;
constexpr int LOAD_WARPS = 16;
constexpr int THREADS = LOAD_WARPS * 32; // 512: four warpgroups
// Shared-memory tile of one operand half (hi or lo): 16 row groups x 8 k chunks of 8 x 16 B core
// matrices.  The cores that are neighbours along K sit 144 bytes apart (128 + 16 of padding),
// so that the 8 lanes which hold one row's eight k chunks store to 8 different bank groups.
constexpr int CORE_K_BYTES = 144;                          // "leading" byte offset
constexpr int CORE_MN_BYTES = 8 * CORE_K_BYTES;            // "stride" byte offset (8-row groups)
constexpr int TILE_BYTES = (BM / 8) * CORE_MN_BYTES;       // 18 KB
constexpr int STAGE_BYTES = 4 * TILE_BYTES;                // A_hi A_lo B_hi B_lo
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;    // 217 KB of the 227 KB a block may use

enum { MODE_K_MAJOR = 0, MODE_MN_MAJOR = 1, MODE_GATHER = 2 };

struct Operand {
    const void *p; // float, or uint8_t when u8
    int mode;
    int ld, vec;   // dense modes: leading dimension, 16-byte loads allowed
    // gather mode (see the header comment); k tables are padded to a multiple of 32 entries
    const int *row_off, *row_yx; // element offset; y | x << 16 (NULL: no coordinates)
    const int *k_off, *k_yx;     // element offset; dy | dx << 16, int16 each
    int y_limit, x_limit;
    int along_k;         // consecutive lanes walk k (else rows)
    int u8;
    float scale;
};

struct GemmArgs {
    Operand A, B;
    const float *bias;
    int bias_vec;        // bias is 16-byte aligned: the dense epilogue may read it as float4
    float *C;            // final output (splits == 1) ...
    float *partial;      // ... or [splits][M][N] partial sums
    const int *c_row_tab; // scatter: C[m, n] at c_row_tab[m] + n * c_col_stride
    int c_col_stride;
    int M, N, K;
    int ldc, c_vec;
    int bn;              // N tile: 32, 64 or 128
    int splits, kb_per_split;
    int relu;
    unsigned long long *times; // debug (B2RL_GEMM_TIMES): 8 %globaltimer stamps per CTA, or NULL
};

__device__ __forceinline__ void stamp(const GemmArgs &g, int slot)
{
    if (g.times) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        g.times[(size_t)blockIdx.x * 8 + slot] = t;
    }
}

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return (uint32_t)__cvta_generic_to_shared(p);
}

// 64-bit wgmma shared-memory matrix descriptor, no swizzle ("interleave", layout type 0): start
// address, the byte offset between the core matrices that are neighbours along K (leading) and
// along M/N (stride), all in 16-byte units.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lead_bytes,
                                              uint32_t stride_bytes)
{
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lead_bytes >> 4) << 16) |
           ((uint64_t)(stride_bytes >> 4) << 32);
}

__device__ __forceinline__ void wgmma_fence()
{
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}

__device__ __forceinline__ void wgmma_commit()
{
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}

template <int N> __device__ __forceinline__ void wgmma_wait()
{
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// Keeps the compiler from moving accesses of an accumulator register across the asynchronous
// wgmma that writes it.
__device__ __forceinline__ void fence_reg(float &r) { asm volatile("" : "+f"(r)::"memory"); }

// D[64 x N] += A[64 x 8] . B[N x 8]^T, tf32 operands from shared memory, f32 accumulators in
// registers: d[4 j + 2 i + c] is row 16 (warp % 4) + lane / 4 + 8 i, column 8 j + 2 (lane % 4) + c.
template <int N> struct Wgmma;

template <> struct Wgmma<16> {
    static __device__ __forceinline__ void mma(float (&d)[8], uint64_t da, uint64_t db)
    {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
                     "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "l"(da), "l"(db), "r"(1));
    }
};

template <> struct Wgmma<32> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t da, uint64_t db)
    {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
                     "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(da), "l"(db), "r"(1));
    }
};

template <> struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db)
    {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
                     "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(da), "l"(db), "r"(1));
    }
};

// x = hi + lo (+ <= 2^-22 |x|), both exactly representable in TF32 (10-bit mantissa, low 13
// bits zero); rounding to nearest in integer arithmetic on the sign-magnitude bit pattern
// (plain integer instructions instead of the conversion pipe).  x - hi is exact.  Inf and
// most NaNs give non-finite results (Inf gives hi = Inf and, through x - hi, a zero lo).  A NaN
// whose leading mantissa bits are all set (0x7fffffff, the NaN CUDA's arithmetic produces) does
// not: the rounding carry runs into the sign bit and leaves hi = lo = -0, so it drops out of
// the product.  Testing every element for it costs 5-7% of the product time on an H100.
__device__ __forceinline__ void split_tf32(float x, uint32_t &hi, uint32_t &lo)
{
    hi = (__float_as_uint(x) + 0x1000u) & 0xffffe000u;
    lo = (__float_as_uint(x - __uint_as_float(hi)) + 0x1000u) & 0xffffe000u;
}

// Four consecutive floats from p (n_valid of them exist), zeros elsewhere.
__device__ __forceinline__ float4 load4(const float *p, bool row_ok, int n_valid, bool vec)
{
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!row_ok || n_valid <= 0) return v;
    if (vec && n_valid >= 4) return __ldg(reinterpret_cast<const float4 *>(p));
    v.x = __ldg(p);
    if (n_valid > 1) v.y = __ldg(p + 1);
    if (n_valid > 2) v.z = __ldg(p + 2);
    if (n_valid > 3) v.w = __ldg(p + 3);
    return v;
}

// One operand tile of one stage: 128 (M or N) x 32 (K) floats, stored K-major: core matrix
// (rg, kc) = rows 8 rg .. 8 rg + 7, k 4 kc .. 4 kc + 3.  Each loader thread owns two 16-byte
// vectors (4 consecutive k of one row) per operand and stage, in one of two lane arrangements:
//   along k   : unit u = rows 4u .. 4u+3 x all 32 k; lanes 8r .. 8r+7 hold row r (a whole
//               128-byte row per 8 lanes: 4 L1 wavefronts per 16-byte load instruction).
//   along rows: unit u = 32 rows x 4 k; lane = row (each warp load instruction is one coalesced
//               run along M/N); the four k values of a thread meet in its 16-byte store -- this
//               is the transposition of the MN-major operands.
struct Frag {
    float4 v[2];
};

template <int MODE> struct Lane { // per thread and operand, fixed for the whole tile
    const float *q[2]; // dense modes: address of this thread's element of k block 0
    int roff[2], ryx[2]; // gather: row table entries
    int tko[2], tkc[2];  // gather: k table entries of two k blocks in flight, lane = k mod 32
    int kofs[2];       // k offset of the thread's vector inside a k block
    int soff[2];       // byte offset of its 16-byte slot inside a tile half, -1: nothing to do
    bool along_k;
};

template <int MODE>
__device__ __forceinline__ void lane_setup(const Operand &o, int mn0, int mn_total, int tile_rows,
                                           int k_first, int lw, int lane, Lane<MODE> &L)
{
    L.along_k = MODE == MODE_K_MAJOR || (MODE == MODE_GATHER && o.along_k);
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int u = lw + 16 * i; // 32 units per tile
        int r, kc;
        if (L.along_k) {
            r = 4 * u + (lane >> 3), kc = lane & 7;
        } else {
            r = (u & 3) * 32 + lane, kc = u >> 2;
        }
        L.kofs[i] = kc * 4;
        // rows past the N tile are never read by the tensor core; rows past the matrix are zero
        L.soff[i] = r < tile_rows ? (r >> 3) * CORE_MN_BYTES + kc * CORE_K_BYTES + (r & 7) * 16
                                  : -1;
        const bool ok = r < tile_rows && mn0 + r < mn_total;
        L.q[i] = nullptr;
        L.roff[i] = L.ryx[i] = 0;
        if (!ok) continue;
        if (MODE == MODE_K_MAJOR)
            L.q[i] = (const float *)o.p + (size_t)(mn0 + r) * o.ld + k_first + kc * 4;
        else if (MODE == MODE_MN_MAJOR)
            L.q[i] = (const float *)o.p + (size_t)(k_first + kc * 4) * o.ld + mn0 + r;
        else {
            L.q[i] = (const float *)o.p; // (marks the row as present)
            L.roff[i] = __ldg(o.row_off + mn0 + r);
            if (o.row_yx) L.ryx[i] = __ldg(o.row_yx + mn0 + r);
        }
    }
}

__device__ __forceinline__ float gather_load(const Operand &o, int idx)
{
    if (o.u8) return (float)__ldg((const uint8_t *)o.p + idx) * o.scale;
    return __ldg((const float *)o.p + idx);
}

// k table entries of one k block -> one register per lane (coalesced; the tables are padded to
// a multiple of 32).  Issued one iteration before the data loads that need them, so that the
// gather is not a chain of two dependent global loads.
template <int MODE>
__device__ __forceinline__ void table_fetch(const Operand &o, Lane<MODE> &L, int slot, int k0,
                                            int lane)
{
    if (MODE != MODE_GATHER) return;
    // the slot is a runtime value: selected, not indexed, so that the tables stay in registers
    const int ko = __ldg(o.k_off + k0 + lane), kc = o.k_yx ? __ldg(o.k_yx + k0 + lane) : 0;
    if (slot) L.tko[1] = ko, L.tkc[1] = kc;
    else L.tko[0] = ko, L.tkc[0] = kc;
}

// Four consecutive k (block-relative kofs .. kofs + 3) of one row; `n` = how many of them lie
// inside K.  All lanes take part in the shuffles, `present` says whether this lane has a row.
__device__ __forceinline__ float4 gather4(const Operand &o, bool present, int roff, int ryx,
                                          int tko, int tkc, int kofs, int n)
{
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    int4 ko;
    ko.x = __shfl_sync(0xffffffffu, tko, kofs);
    ko.y = __shfl_sync(0xffffffffu, tko, kofs + 1);
    ko.z = __shfl_sync(0xffffffffu, tko, kofs + 2);
    ko.w = __shfl_sync(0xffffffffu, tko, kofs + 3);
    if (o.row_yx == nullptr) {
        if (!present || n <= 0) return v;
        v.x = gather_load(o, roff + ko.x);
        if (n > 1) v.y = gather_load(o, roff + ko.y);
        if (n > 2) v.z = gather_load(o, roff + ko.z);
        if (n > 3) v.w = gather_load(o, roff + ko.w);
        return v;
    }
    int4 kc;
    kc.x = __shfl_sync(0xffffffffu, tkc, kofs);
    kc.y = __shfl_sync(0xffffffffu, tkc, kofs + 1);
    kc.z = __shfl_sync(0xffffffffu, tkc, kofs + 2);
    kc.w = __shfl_sync(0xffffffffu, tkc, kofs + 3);
    if (!present || n <= 0) return v;
    const int ry = ryx & 0xffff, rx = ryx >> 16;
    const unsigned yl = (unsigned)o.y_limit, xl = (unsigned)o.x_limit;
#define B2RL_OK_AT(c) \
    ((unsigned)(ry + (int)(short)((c) & 0xffff)) < yl && (unsigned)(rx + ((c) >> 16)) < xl)
    if (B2RL_OK_AT(kc.x)) v.x = gather_load(o, roff + ko.x);
    if (n > 1 && B2RL_OK_AT(kc.y)) v.y = gather_load(o, roff + ko.y);
    if (n > 2 && B2RL_OK_AT(kc.z)) v.z = gather_load(o, roff + ko.z);
    if (n > 3 && B2RL_OK_AT(kc.w)) v.w = gather_load(o, roff + ko.w);
#undef B2RL_OK_AT
    return v;
}

// k block `kb` (relative to the first one of this CTA) -> registers.  `full`: the whole block
// lies inside K (warp-uniform), which is the common case and needs no per-element checks.
template <int MODE>
__device__ __forceinline__ void fetch_operand(const Operand &o, const Lane<MODE> &L, int kb,
                                              int slot, int k0, int k_total, Frag &f)
{
    const bool full = k0 + BK <= k_total;
#pragma unroll
    for (int i = 0; i < 2; i++) {
        if (MODE == MODE_GATHER) {
            f.v[i] = gather4(o, L.q[i] != nullptr, L.roff[i], L.ryx[i],
                             slot ? L.tko[1] : L.tko[0], slot ? L.tkc[1] : L.tkc[0],
                             L.kofs[i], full ? 4 : k_total - (k0 + L.kofs[i]));
            continue;
        }
        f.v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (L.q[i] == nullptr) continue;
        if (MODE == MODE_K_MAJOR) {
            const float *q = L.q[i] + (size_t)kb * BK;
            if (full && o.vec)
                f.v[i] = __ldg(reinterpret_cast<const float4 *>(q));
            else
                f.v[i] = load4(q, true, k_total - (k0 + L.kofs[i]), o.vec);
        } else {
            const float *q = L.q[i] + (size_t)kb * BK * o.ld;
            const int left = k_total - (k0 + L.kofs[i]);
            if (full || left > 0) f.v[i].x = __ldg(q);
            if (full || left > 1) f.v[i].y = __ldg(q + o.ld);
            if (full || left > 2) f.v[i].z = __ldg(q + 2 * (size_t)o.ld);
            if (full || left > 3) f.v[i].w = __ldg(q + 3 * (size_t)o.ld);
        }
    }
}

template <int MODE>
__device__ __forceinline__ void store_operand(const Lane<MODE> &L, const Frag &f, uint8_t *s_hi,
                                              uint8_t *s_lo)
{
#pragma unroll
    for (int i = 0; i < 2; i++) {
        if (L.soff[i] < 0) continue;
        uint4 h, l;
        split_tf32(f.v[i].x, h.x, l.x);
        split_tf32(f.v[i].y, h.y, l.y);
        split_tf32(f.v[i].z, h.z, l.z);
        split_tf32(f.v[i].w, h.w, l.w);
        *reinterpret_cast<uint4 *>(s_hi + L.soff[i]) = h;
        *reinterpret_cast<uint4 *>(s_lo + L.soff[i]) = l;
    }
}

template <int AMODE, int BMODE, int TBN>
__global__ void __launch_bounds__(THREADS, 1) k_gemm_tf32x3(const __grid_constant__ GemmArgs g)
{
    constexpr int WN = TBN / 2;  // columns of one warpgroup's quadrant
    constexpr int NACC = WN / 2; // registers per thread of one 64 x WN accumulator
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    const int tiles_n = (g.N + TBN - 1) / TBN;
    const int tile = blockIdx.x / g.splits, split = blockIdx.x % g.splits;
    const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * TBN;
    const int kb_total = (g.K + BK - 1) / BK;
    const int kb0 = split * g.kb_per_split;
    const int kb1 = min(kb_total, kb0 + g.kb_per_split);
    const int n_kb = kb1 - kb0; // >= 1 by construction of the launch

    if (threadIdx.x == 0) stamp(g, 0);
    Lane<AMODE> la;
    Lane<BMODE> lb;
    lane_setup<AMODE>(g.A, m0, g.M, BM, kb0 * BK, warp, lane, la);
    lane_setup<BMODE>(g.B, n0, g.N, TBN, kb0 * BK, warp, lane, lb);
    if (threadIdx.x == 0) stamp(g, 1); // set-up done

    // the quadrant of this warpgroup: rows wm .. wm + 63, columns wn .. wn + WN - 1 of the tile
    const int wm = (wg & 1) * 64, wn = (wg >> 1) * WN;
    const uint32_t a_off = (wm / 8) * CORE_MN_BYTES, b_off = (wn / 8) * CORE_MN_BYTES;
    // the two correction products have their own accumulator: the tensor core truncates on
    // every accumulation, so the long hi.hi chain should not carry the small terms (and vice
    // versa); the epilogue adds the two
    float acc[NACC], cor[NACC];
#pragma unroll
    for (int i = 0; i < NACC; i++) acc[i] = cor[i] = 0.f;

    // The table entries of k block i + 2 and the data of k block i + 1 are fetched while the
    // tensor cores work on block i.
    Frag fa, fb;
    table_fetch<AMODE>(g.A, la, 0, kb0 * BK, lane);
    table_fetch<BMODE>(g.B, lb, 0, kb0 * BK, lane);
    if (n_kb > 1) {
        table_fetch<AMODE>(g.A, la, 1, (kb0 + 1) * BK, lane);
        table_fetch<BMODE>(g.B, lb, 1, (kb0 + 1) * BK, lane);
    }
    fetch_operand<AMODE>(g.A, la, 0, 0, kb0 * BK, g.K, fa);
    fetch_operand<BMODE>(g.B, lb, 0, 0, kb0 * BK, g.K, fb);
    for (int it = 0; it < n_kb; it++) {
        const int s = it % STAGES;
        uint8_t *st = smem + s * STAGE_BYTES;
        // stage s was last read by the wgmma of block it - 3, which every warpgroup waited for
        // (wait_group 1 at it - 2) before it arrived at the barrier of block it - 1
        store_operand<AMODE>(la, fa, st, st + TILE_BYTES);
        store_operand<BMODE>(lb, fb, st + 2 * TILE_BYTES, st + 3 * TILE_BYTES);
        // generic-proxy stores -> visible to the tensor core (async proxy)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (it == 0 && threadIdx.x == 0) stamp(g, 2); // first stage filled
        if (it + 1 < n_kb) {
            const int k1 = (kb0 + it + 1) * BK;
            fetch_operand<AMODE>(g.A, la, it + 1, (it + 1) & 1, k1, g.K, fa);
            fetch_operand<BMODE>(g.B, lb, it + 1, (it + 1) & 1, k1, g.K, fb);
            if (it + 2 < n_kb) { // table slot it & 1 belonged to block `it`, whose loads are out
                table_fetch<AMODE>(g.A, la, it & 1, (kb0 + it + 2) * BK, lane);
                table_fetch<BMODE>(g.B, lb, it & 1, (kb0 + it + 2) * BK, lane);
            }
        }
        const uint32_t sa = smem_u32(st) + a_off, sb = smem_u32(st) + 2 * TILE_BYTES + b_off;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < BK / 8; j++) {
            // one k step = two k chunks: neighbours along K 144 B apart, 8-row groups 1152 B
            const uint32_t step = j * 2 * CORE_K_BYTES;
            const uint64_t a_hi = make_desc(sa + step, CORE_K_BYTES, CORE_MN_BYTES);
            const uint64_t a_lo = make_desc(sa + TILE_BYTES + step, CORE_K_BYTES, CORE_MN_BYTES);
            const uint64_t b_hi = make_desc(sb + step, CORE_K_BYTES, CORE_MN_BYTES);
            const uint64_t b_lo = make_desc(sb + TILE_BYTES + step, CORE_K_BYTES, CORE_MN_BYTES);
            Wgmma<WN>::mma(cor, a_lo, b_hi);
            Wgmma<WN>::mma(cor, a_hi, b_lo);
            Wgmma<WN>::mma(acc, a_hi, b_hi);
        }
        wgmma_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < NACC; i++) fence_reg(acc[i]), fence_reg(cor[i]);
    if (threadIdx.x == 0) stamp(g, 3); // this warpgroup's products complete

    // ---------------- epilogue: the tile goes through shared memory (the operand ring is idle
    // once every warpgroup is past its last wait) as [128][bn + 4] floats ----------------
    __syncthreads();
    if (threadIdx.x == 0) stamp(g, 4); // accumulators complete
    constexpr int SROW = TBN + 4;
    float *stage_tile = reinterpret_cast<float *>(smem);
    {
        const int r0 = wm + 16 * (warp & 3) + (lane >> 2), c0 = wn + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < WN / 8; j++)
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int d = 4 * j + 2 * i;
                *reinterpret_cast<float2 *>(stage_tile + (r0 + 8 * i) * SROW + c0 + 8 * j) =
                    make_float2(acc[d] + cor[d], acc[d + 1] + cor[d + 1]);
            }
    }
    __syncthreads();
    const bool direct = g.splits == 1;
    const bool scatter = direct && g.c_row_tab != nullptr;
    float *out = direct ? g.C : g.partial + (size_t)split * g.M * g.N;
    const int ldo = direct ? g.ldc : g.N;
    const bool vec = direct ? g.c_vec : (g.N % 4 == 0);
    const bool bias_relu = direct;
    const int t = threadIdx.x;
    if (scatter) {
        // NCHW activations / transposed weight gradients: C[m, n] at c_row_tab[m] + n * stride;
        // consecutive threads take consecutive rows (one coalesced run per column)
        for (int idx = t; idx < BM * TBN; idx += THREADS) {
            const int rr = idx % BM, cc = idx / BM;
            if (m0 + rr >= g.M || n0 + cc >= g.N) continue;
            float y = stage_tile[rr * SROW + cc];
            if (g.bias) y += __ldg(g.bias + n0 + cc);
            if (g.relu) y = fmaxf(y, 0.f);
            out[(long long)__ldg(g.c_row_tab + m0 + rr) + (long long)(n0 + cc) * g.c_col_stride] = y;
        }
    } else if (vec && (n0 & 3) == 0) {
        const int per_row = TBN / 4;
        for (int idx = t; idx < BM * per_row; idx += THREADS) {
            const int rr = idx / per_row, cc = (idx % per_row) * 4;
            if (m0 + rr >= g.M || n0 + cc >= g.N) continue;
            float4 x = *reinterpret_cast<const float4 *>(stage_tile + rr * SROW + cc);
            float *o = out + (size_t)(m0 + rr) * ldo + n0 + cc;
            if (n0 + cc + 4 <= g.N) {
                if (bias_relu && g.bias) {
                    const float *bp = g.bias + n0 + cc;
                    const float4 bv = g.bias_vec
                                          ? __ldg(reinterpret_cast<const float4 *>(bp))
                                          : make_float4(__ldg(bp), __ldg(bp + 1), __ldg(bp + 2),
                                                        __ldg(bp + 3));
                    x.x += bv.x, x.y += bv.y, x.z += bv.z, x.w += bv.w;
                }
                if (bias_relu && g.relu)
                    x.x = fmaxf(x.x, 0.f), x.y = fmaxf(x.y, 0.f), x.z = fmaxf(x.z, 0.f),
                    x.w = fmaxf(x.w, 0.f);
                *reinterpret_cast<float4 *>(o) = x;
            } else {
                const float xs[4] = {x.x, x.y, x.z, x.w};
                for (int j = 0; j < 4 && n0 + cc + j < g.N; j++) {
                    float y = xs[j];
                    if (bias_relu && g.bias) y += __ldg(g.bias + n0 + cc + j);
                    if (bias_relu && g.relu) y = fmaxf(y, 0.f);
                    o[j] = y;
                }
            }
        }
    } else {
        for (int idx = t; idx < BM * TBN; idx += THREADS) {
            const int rr = idx / TBN, cc = idx % TBN;
            if (m0 + rr >= g.M || n0 + cc >= g.N) continue;
            float y = stage_tile[rr * SROW + cc];
            if (bias_relu && g.bias) y += __ldg(g.bias + n0 + cc);
            if (bias_relu && g.relu) y = fmaxf(y, 0.f);
            out[(size_t)(m0 + rr) * ldo + n0 + cc] = y;
        }
    }
    if (threadIdx.x == 0) stamp(g, 5); // epilogue stores issued
    __syncthreads();
    if (threadIdx.x == 0) stamp(g, 6);
}

// C = sum over the K splits + bias, relu; dense or scattered like the epilogue.  The order of
// the additions never depends on timing, so results are run-to-run identical.
// Large outputs: one thread per output, splits added in order (coalesced across the threads).
__global__ void __launch_bounds__(256) k_gemm_reduce(const float *__restrict__ partial, int splits,
                                                     int M, int N, const float *__restrict__ bias,
                                                     int relu, float *__restrict__ C, int ldc,
                                                     const int *__restrict__ row_tab,
                                                     int col_stride)
{
    const size_t total = (size_t)M * N;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (size_t)gridDim.x * blockDim.x) {
        float acc = partial[i];
        for (int s = 1; s < splits; s++) acc += partial[(size_t)s * total + i];
        const int m = (int)(i / N), n = (int)(i % N);
        if (bias) acc += __ldg(bias + n);
        if (relu) acc = fmaxf(acc, 0.f);
        if (row_tab)
            C[(long long)__ldg(row_tab + m) + (long long)n * col_stride] = acc;
        else
            C[(size_t)m * ldc + n] = acc;
    }
}

// Small outputs with many splits (the weight gradients: 32 K outputs, 36 splits): a block of
// 8 warps works on 32 consecutive outputs, warp w adds the splits w, w + 8, ... (coalesced
// 128-byte reads), the eight partial sums meet in shared memory and are added in warp order.
__global__ void __launch_bounds__(256) k_gemm_reduce_deep(const float *__restrict__ partial,
                                                          int splits, int M, int N,
                                                          const float *__restrict__ bias, int relu,
                                                          float *__restrict__ C, int ldc,
                                                          const int *__restrict__ row_tab,
                                                          int col_stride)
{
    __shared__ float red[8][32];
    const size_t total = (size_t)M * N;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (size_t base = (size_t)blockIdx.x * 32; base < total; base += (size_t)gridDim.x * 32) {
        const size_t i = base + lane;
        float acc = 0.f;
        if (i < total)
            for (int s = warp; s < splits; s += 8) acc += partial[(size_t)s * total + i];
        red[warp][lane] = acc;
        __syncthreads();
        if (warp == 0 && i < total) {
            acc = red[0][lane];
#pragma unroll
            for (int w = 1; w < 8; w++) acc += red[w][lane];
            const int m = (int)(i / N), n = (int)(i % N);
            if (bias) acc += __ldg(bias + n);
            if (relu) acc = fmaxf(acc, 0.f);
            if (row_tab)
                C[(long long)__ldg(row_tab + m) + (long long)n * col_stride] = acc;
            else
                C[(size_t)m * ldc + n] = acc;
        }
        __syncthreads();
    }
}

int sm_count_cached()
{
    static int sm_count = 0;
    if (!sm_count) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
        if (sm_count <= 0) sm_count = 132;
    }
    return sm_count;
}

int n_tile(int N) { return N <= 32 ? 32 : N <= 64 ? 64 : 128; }

// How the launch cuts the contraction: enough CTAs to cover the SMs, at least 4 k blocks each.
void plan_splits(int M, int N, int K, int *splits, int *kb_per_split)
{
    const int bn = n_tile(N);
    const int tiles = ((M + BM - 1) / BM) * ((N + bn - 1) / bn);
    const int kb = (K + BK - 1) / BK;
    int s = sm_count_cached() / tiles;
    if (s > kb / 4) s = kb / 4;
    if (s < 1) s = 1;
    int per = (kb + s - 1) / s;
    s = (kb + per - 1) / per; // no empty split
    *splits = s;
    *kb_per_split = per;
}

int fill_operand(const b2rl_gemm_operand *src, int rows, int K, Operand *dst, const char *name)
{
    B2RL_REQUIRE(src && src->data, B2RL_ERR_INVALID, "gemm: operand %s is null", name);
    dst->p = src->data;
    dst->mode = src->mode;
    dst->ld = src->ld;
    dst->vec = 0;
    dst->row_off = src->row_off, dst->row_yx = src->row_yx;
    dst->k_off = src->k_off, dst->k_yx = src->k_yx;
    dst->y_limit = src->y_limit, dst->x_limit = src->x_limit;
    dst->along_k = src->lanes_along_k ? 1 : 0;
    dst->u8 = src->u8 ? 1 : 0;
    dst->scale = src->scale;
    switch (src->mode) {
    case B2RL_GEMM_K_MAJOR:
    case B2RL_GEMM_MN_MAJOR:
        B2RL_REQUIRE(!src->u8, B2RL_ERR_INVALID, "gemm: dense operand %s must be fp32", name);
        B2RL_REQUIRE(src->ld >= (src->mode == B2RL_GEMM_K_MAJOR ? K : rows), B2RL_ERR_RANGE,
                     "gemm: leading dimension of %s smaller than its rows", name);
        B2RL_REQUIRE(((uintptr_t)src->data & 3) == 0, B2RL_ERR_INVALID,
                     "gemm: operand %s must be 4-byte aligned", name);
        dst->vec = (((uintptr_t)src->data & 15) == 0 && src->ld % 4 == 0);
        break;
    case B2RL_GEMM_GATHER:
        B2RL_REQUIRE(src->row_off && src->k_off, B2RL_ERR_INVALID,
                     "gemm: gather operand %s needs its row and k offset tables", name);
        B2RL_REQUIRE((src->row_yx == nullptr) == (src->k_yx == nullptr), B2RL_ERR_INVALID,
                     "gemm: gather operand %s: coordinates on both tables or on none", name);
        B2RL_REQUIRE(((uintptr_t)src->k_off & 15) == 0 && ((uintptr_t)src->k_yx & 15) == 0,
                     B2RL_ERR_INVALID, "gemm: k tables of %s must be 16-byte aligned", name);
        B2RL_REQUIRE(!src->row_yx || (src->y_limit > 0 && src->x_limit > 0), B2RL_ERR_RANGE,
                     "gemm: gather limits of %s out of range", name);
        break;
    default:
        B2RL_REQUIRE(false, B2RL_ERR_INVALID, "gemm: unknown operand mode %d", src->mode);
    }
    return B2RL_OK;
}

} // namespace

static unsigned long long *g_gemm_times = nullptr; // debug: set by b2rl_gemm_debug_times

// Debug aid (tools/gemm_phases.py): stamps of the phases of every CTA of the next launches go
// to `device_buffer` (8 x uint64 per CTA, large enough for the largest grid); NULL switches off.
extern "C" int b2rl_gemm_debug_times(void *device_buffer)
{
    g_gemm_times = (unsigned long long *)device_buffer;
    return B2RL_OK;
}

extern "C" int64_t b2rl_gemm_workspace_bytes(int32_t M, int32_t N, int32_t K)
{
    if (M <= 0 || N <= 0 || K <= 0) return 0;
    int splits, per;
    plan_splits(M, N, K, &splits, &per);
    return splits > 1 ? (int64_t)splits * M * N * (int64_t)sizeof(float) : 0;
}

extern "C" int b2rl_gemm_tf32x3_ex(const b2rl_gemm_operand *A, const b2rl_gemm_operand *B,
                                   const b2rl_gemm_output *C, int32_t M, int32_t N, int32_t K,
                                   void *workspace, int64_t workspace_bytes, void *stream)
{
    B2RL_REQUIRE(C && C->data, B2RL_ERR_INVALID, "gemm_tf32x3: null output");
    B2RL_REQUIRE(M > 0 && N > 0 && K > 0, B2RL_ERR_RANGE, "gemm_tf32x3: empty product");
    GemmArgs g;
    int rc = fill_operand(A, M, K, &g.A, "A");
    if (rc != B2RL_OK) return rc;
    rc = fill_operand(B, N, K, &g.B, "B");
    if (rc != B2RL_OK) return rc;
    // a bias that is a view into a larger buffer (a flat parameter vector) may start at any float
    g.bias = C->bias, g.bias_vec = ((uintptr_t)C->bias & 15) == 0, g.C = C->data;
    g.c_row_tab = C->row_tab, g.c_col_stride = C->col_stride;
    B2RL_REQUIRE(C->row_tab || C->ld >= N, B2RL_ERR_RANGE,
                 "gemm_tf32x3: leading dimension of C smaller than its rows");
    B2RL_REQUIRE(((uintptr_t)C->data & 3) == 0 && ((uintptr_t)C->bias & 3) == 0,
                 B2RL_ERR_INVALID, "gemm_tf32x3: C and bias must be 4-byte aligned");
    g.M = M, g.N = N, g.K = K, g.ldc = C->ld;
    g.c_vec = (!C->row_tab && ((uintptr_t)C->data & 15) == 0 && C->ld % 4 == 0);
    g.relu = C->relu ? 1 : 0;
    g.times = g_gemm_times;
    g.bn = n_tile(N);
    plan_splits(M, N, K, &g.splits, &g.kb_per_split);
    g.partial = nullptr;
    if (g.splits > 1) {
        const int64_t need = (int64_t)g.splits * M * N * (int64_t)sizeof(float);
        B2RL_REQUIRE(workspace && workspace_bytes >= need && ((uintptr_t)workspace & 15) == 0,
                     B2RL_ERR_INVALID,
                     "gemm_tf32x3: workspace of %lld bytes (16-byte aligned) required",
                     (long long)need);
        g.partial = (float *)workspace;
    }
    typedef void (*kernel_t)(GemmArgs);
#define B2RL_GEMM_BN(a, b) {k_gemm_tf32x3<a, b, 32>, k_gemm_tf32x3<a, b, 64>, k_gemm_tf32x3<a, b, 128>}
#define B2RL_GEMM_B(a) {B2RL_GEMM_BN(a, 0), B2RL_GEMM_BN(a, 1), B2RL_GEMM_BN(a, 2)}
    static const kernel_t kernels[3][3][3] = {B2RL_GEMM_B(0), B2RL_GEMM_B(1), B2RL_GEMM_B(2)};
#undef B2RL_GEMM_B
#undef B2RL_GEMM_BN
    const int bi = g.bn == 32 ? 0 : g.bn == 64 ? 1 : 2;
    const kernel_t kernel = kernels[g.A.mode][g.B.mode][bi];
    static bool attr_set[64][3][3][3]; // per device and instantiation
    int cur_dev = 0;
    B2RL_CUDA(cudaGetDevice(&cur_dev));
    if (cur_dev < 0 || cur_dev >= 64 || !attr_set[cur_dev][g.A.mode][g.B.mode][bi]) {
        B2RL_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SMEM_BYTES));
        if (cur_dev >= 0 && cur_dev < 64) attr_set[cur_dev][g.A.mode][g.B.mode][bi] = true;
    }
    const int tiles = ((M + BM - 1) / BM) * ((N + g.bn - 1) / g.bn);
    kernel<<<tiles * g.splits, THREADS, SMEM_BYTES, (cudaStream_t)stream>>>(g);
    B2RL_CUDA(cudaGetLastError());
    if (g.splits > 1) {
        const long long total = (long long)M * N;
        if (total >= 65536 || g.splits <= 8) {
            long long blocks = (total + 255) / 256;
            if (blocks > 8ll * sm_count_cached()) blocks = 8ll * sm_count_cached();
            k_gemm_reduce<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(
                g.partial, g.splits, M, N, C->bias, g.relu, C->data, C->ld, C->row_tab,
                C->col_stride);
        } else {
            long long blocks = (total + 31) / 32;
            if (blocks > 8ll * sm_count_cached()) blocks = 8ll * sm_count_cached();
            k_gemm_reduce_deep<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(
                g.partial, g.splits, M, N, C->bias, g.relu, C->data, C->ld, C->row_tab,
                C->col_stride);
        }
        B2RL_CUDA(cudaGetLastError());
    }
    return B2RL_OK;
}

extern "C" int b2rl_gemm_tf32x3(const float *A, int32_t lda, int32_t a_mn_major, const float *B,
                                int32_t ldb, int32_t b_mn_major, const float *bias, int32_t relu,
                                float *C, int32_t ldc, int32_t M, int32_t N, int32_t K,
                                void *workspace, int64_t workspace_bytes, void *stream)
{
    b2rl_gemm_operand a, b;
    b2rl_gemm_output c;
    memset(&a, 0, sizeof a), memset(&b, 0, sizeof b), memset(&c, 0, sizeof c);
    a.data = A, a.ld = lda, a.mode = a_mn_major ? B2RL_GEMM_MN_MAJOR : B2RL_GEMM_K_MAJOR;
    b.data = B, b.ld = ldb, b.mode = b_mn_major ? B2RL_GEMM_MN_MAJOR : B2RL_GEMM_K_MAJOR;
    c.data = C, c.ld = ldc, c.bias = bias, c.relu = relu;
    return b2rl_gemm_tf32x3_ex(&a, &b, &c, M, N, K, workspace, workspace_bytes, stream);
}
