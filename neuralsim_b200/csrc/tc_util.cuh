// Hopper tensor-core plumbing used by the fused MLP kernels: warpgroup MMAs (wgmma) with both operands in shared memory
// and fp32 accumulators in registers.  Inline PTX only (no CUTLASS dependency).  Every kernel that uses it runs one
// warpgroup (128 threads) per CTA; the MMA helpers are collective over it and must be reached by all 128 threads.
//
// Shared-memory operand layout ("canonical K-major, no swizzle", what cute calls Layout_K_INTER_Atom):
//   the tile is cut into core matrices of 8 rows x 16 bytes (8 fp16 along K); a core matrix is 128 contiguous
//   bytes (row r at r*16).  SBO = byte distance between core matrices that are adjacent along M/N (next 8 rows),
//   LBO = byte distance between core matrices that are adjacent along K (next 8 k).
//   We store a [R x K] fp16 tile chunk-major:   byte(r, k) = (k/8) * (R*16) + r*16 + (k%8)*2
//   => SBO = 128, LBO = R*16.  Thread r owns row r and writes K/8 16-byte vectors with a stride of R*16 bytes:
//   consecutive threads hit consecutive 16-byte slots, i.e. conflict-free st.shared.v4.
//   The very same bytes read as an MN-major (transposed) operand (rows <-> K) are described by swapping the two
//   offsets (LBO = 128, SBO = R*16) -- used by the weight-gradient MMAs that contract over the points of a tile.
//
// A 128-row tile is two m64 wgmma row blocks.  The accumulator of rows [64h, 64h + 64) lives in d[h][] in the wgmma
// fragment layout: warp w, lane l holds rows 64h + 16w + l/4 (+8) and columns 8c + 2(l%4) (+1).  Kernels whose
// epilogue wants "thread r owns row r" stage the fragments in a padded fp32 row buffer in shared memory (frag_store,
// then a CTA barrier, then acc_ld8 of the own row).
#pragma once
#include "nsb_common.cuh"

namespace nsb {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 64-bit wgmma shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor):
//   [0,14) start address >> 4 | [16,30) LBO >> 4 | [32,46) SBO >> 4 | [49,52) base offset = 0 | [62,64) swizzle = 0 (none)
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}

// One chunk-major fp16 tile in shared memory as an MMA operand; kstep = bytes between consecutive K = 16 slices.
struct Operand {
    uint32_t addr, lbo, sbo, kstep;
};
// a [rows x K] tile contracted over its columns (K-major)
__device__ __forceinline__ Operand kmajor(uint32_t addr, int rows) { return Operand{addr, (uint32_t)rows * 16, 128, (uint32_t)rows * 32}; }
// the same bytes contracted over its rows (MN-major: K = the rows, M or N = the columns)
__device__ __forceinline__ Operand mnmajor(uint32_t addr, int rows) { return Operand{addr, 128, (uint32_t)rows * 16, 256}; }

// wgmma.mma_async m64nNk16, fp16 x fp16 -> fp32, A and B from shared memory; TA / TB = 1: the operand is MN-major.
template <int N, int TA, int TB>
struct Wgmma;
template <int TA, int TB>
struct Wgmma<32, TA, TB> {
    __device__ __forceinline__ static void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB>
struct Wgmma<40, TA, TB> {
    __device__ __forceinline__ static void mma(float (&d)[20], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %22, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n40k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, %20, %21, p, 1, 1, %23, %24;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
            : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB>
struct Wgmma<48, TA, TB> {
    __device__ __forceinline__ static void mma(float (&d)[24], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, %27, %28;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB>
struct Wgmma<64, TA, TB> {
    __device__ __forceinline__ static void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <int TA, int TB>
struct Wgmma<80, TA, TB> {
    __device__ __forceinline__ static void mma(float (&d)[40], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, %43, %44;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
            : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of an accumulator register across the asynchronous MMA
__device__ __forceinline__ void fence_operand(float &r) { asm volatile("" : "+f"(r)::"memory"); }

// D[128 x N] (+)= A[128 x 16 KSTEPS] . B[16 KSTEPS x N] by the whole warpgroup; returns when the result is in d.
// The shared-memory operands must have been made visible to the async proxy (fence_async_smem + barrier) before.
template <int N, int TA, int TB, int KSTEPS>
__device__ __forceinline__ void mma_m128(float (&d)[2][N / 2], const Operand &a, const Operand &b, bool accumulate) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) fence_operand(d[h][i]);
    wgmma_fence();
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int ks = 0; ks < KSTEPS; ++ks)
            Wgmma<N, TA, TB>::mma(d[h], make_desc(a.addr + h * 8 * a.sbo + ks * a.kstep, a.lbo, a.sbo), make_desc(b.addr + ks * b.kstep, b.lbo, b.sbo),
                                  (ks > 0 || accumulate) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait_all();
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) fence_operand(d[h][i]);
}

// Row buffer of staged accumulators: row r at acc + r * stride (floats).  A stride = 4 (mod 8) keeps the row reads of
// acc_ld8 free of bank conflicts.
constexpr int acc_stride(int cols) { return cols + 4; }

// this thread's fragments of D[128 x N] -> columns [col0, col0 + N) of the row buffer (fp32, exact)
template <int N>
__device__ __forceinline__ void frag_store(const float (&d)[2][N / 2], float *acc, int stride, int col0) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int c = 0; c < N / 8; ++c)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int row = h * 64 + w * 16 + (l >> 2) + 8 * i, col = col0 + c * 8 + 2 * (l & 3);
                *reinterpret_cast<float2 *>(acc + row * stride + col) = make_float2(d[h][4 * c + 2 * i], d[h][4 * c + 2 * i + 1]);
            }
}
template <int N>
__device__ __forceinline__ void frag_load(float (&d)[2][N / 2], const float *acc, int stride, int col0) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int c = 0; c < N / 8; ++c)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int row = h * 64 + w * 16 + (l >> 2) + 8 * i, col = col0 + c * 8 + 2 * (l & 3);
                const float2 v = *reinterpret_cast<const float2 *>(acc + row * stride + col);
                d[h][4 * c + 2 * i] = v.x;
                d[h][4 * c + 2 * i + 1] = v.y;
            }
}
// D[128 x N] (+)= A . B with D kept in columns [col0, col0 + N) of the row buffer: load (if accumulating), MMA, store.
// Only this thread's own fragment positions are read and written; the rows are readable by their owners after a barrier.
template <int N, int TA, int TB, int KSTEPS>
__device__ __forceinline__ void mma_to_rows(float *acc, int stride, int col0, const Operand &a, const Operand &b, bool accumulate) {
    float d[2][N / 2];
    if (accumulate) frag_load<N>(d, acc, stride, col0);
    else {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < N / 2; ++i) d[h][i] = 0.f;
    }
    mma_m128<N, TA, TB, KSTEPS>(d, a, b, accumulate);
    frag_store<N>(d, acc, stride, col0);
}

// 8 consecutive staged fp32 columns of one row
__device__ __forceinline__ void acc_ld8(const float *acc, int stride, int row, int col, float (&v)[8]) {
    const float4 a = *reinterpret_cast<const float4 *>(acc + row * stride + col), b = *reinterpret_cast<const float4 *>(acc + row * stride + col + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tWAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// ---- TMA (bulk async copy engine): one thread moves `bytes` contiguous bytes global -> shared; completion is counted on an mbarrier.
//      bytes % 16 == 0, both addresses 16-byte aligned.  The issuing thread first announces the byte count (arrive.expect_tx).
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_bulk(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gmem_src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ uint4 pack8_f16(const float (&v)[8]) {
    __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
    __half2 h2 = __floats2half2_rn(v[4], v[5]), h3 = __floats2half2_rn(v[6], v[7]);
    uint4 q;
    q.x = *reinterpret_cast<uint32_t *>(&h0); q.y = *reinterpret_cast<uint32_t *>(&h1);
    q.z = *reinterpret_cast<uint32_t *>(&h2); q.w = *reinterpret_cast<uint32_t *>(&h3);
    return q;
}

// write one row of a chunk-major [R x K] fp16 tile: `vals` are K fp32 values rounded to fp16 here
template <int R, int K>
__device__ __forceinline__ void store_row_f16(uint8_t *tile, int r, const float *vals) {
#pragma unroll
    for (int c = 0; c < K / 8; ++c) {
        __half2 h0 = __floats2half2_rn(vals[c * 8 + 0], vals[c * 8 + 1]);
        __half2 h1 = __floats2half2_rn(vals[c * 8 + 2], vals[c * 8 + 3]);
        __half2 h2 = __floats2half2_rn(vals[c * 8 + 4], vals[c * 8 + 5]);
        __half2 h3 = __floats2half2_rn(vals[c * 8 + 6], vals[c * 8 + 7]);
        uint4 q;
        q.x = *reinterpret_cast<uint32_t *>(&h0);
        q.y = *reinterpret_cast<uint32_t *>(&h1);
        q.z = *reinterpret_cast<uint32_t *>(&h2);
        q.w = *reinterpret_cast<uint32_t *>(&h3);
        *reinterpret_cast<uint4 *>(tile + c * (R * 16) + r * 16) = q;
    }
}

}  // namespace tc
}  // namespace nsb
