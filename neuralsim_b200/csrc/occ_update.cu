// The occupancy grid's update from the network on the device (OccGridEma.step's body, fields/occ_update.py), sm_90a.
//
// Reference: OccGridEma._step (nr3d_lib/models/accelerations/occgrid/ema_single.py:133-175) + sample_pts_in_voxels (occgrid/utils.py:17-41):
//   occupied, empty = occ_grid.nonzero(), (~occ_grid).nonzero()                     two host reads
//   num_steps times:  warm-up:  sample_pts_in_voxels(all cells, num_pts)
//                     else:     all cells num_pts // 2, empty num_pts // 4 (if any), occupied num_pts // 4 (asserts there are some)
//   sample_pts_in_voxels(gidx, n):  n < 2 nv:  vidx = randint(nv, [n]); off = rand([n, 3]); pts = ((gidx[vidx] + off) / res) * 2 - 1
//                                   else:      per = n // nv + 1; off = rand([nv, per, 3]); pts = ((gidx[:, None] + off) / res) * 2 - 1
// Here the two lists come from one scan of the grid (nsb_scan_counts: the occupied cells in order, and the exclusive count of occupied
// cells before every cell, which places the empty ones), their sizes stay on the device, and ONE kernel draws every point of the
// num_steps iterations: each thread rebuilds the (at most three) parts of an iteration from the device counts, finds the part of its
// point and the Philox offset of that part's draws (base + the inc() of every draw before it, torch_uniform.cuh), and evaluates torch's
// values and roundings element by element.
#include "torch_uniform.cuh"

namespace nsb {

__global__ void __launch_bounds__(256) k_occ_flags(const uint8_t *__restrict__ occ, int64_t cells, int32_t *__restrict__ flags) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < cells; c += (int64_t)gridDim.x * blockDim.x) flags[c] = occ[c] ? 1 : 0;
}

// empty[c - first[c]] = c for every empty cell (first = occupied cells before c); counts[1] = the number of empty cells
__global__ void __launch_bounds__(256)
k_occ_empty_list(const int32_t *__restrict__ flags, const int32_t *__restrict__ first, int64_t cells, int64_t *__restrict__ empty,
                 int64_t *__restrict__ counts) {
    const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i0 == 0) counts[1] = cells - counts[0];
    for (int64_t c = i0; c < cells; c += (int64_t)gridDim.x * blockDim.x)
        if (!flags[c]) empty[c - first[c]] = c;
}

// one sample_pts_in_voxels call: nv listed voxels (list NULL: every cell, in order), n points asked for
struct OccPart {
    const int64_t *list;
    int64_t nv, n, per, npts, first_pt;     // per > 0: the n_per_vox branch
    uint64_t first_off;                     // offset of its first draw, relative to the iteration's
};

struct OccIter {
    OccPart p[3];
    int np;
    int64_t pts;                            // points of one iteration
    uint64_t inc;                           // generator offsets of one iteration
    bool empty_occupied;                    // the steady phase with no occupied voxel: nothing is drawn (the reference asserts)
};

__device__ __forceinline__ void occ_add_part(OccIter &it, const int64_t *list, int64_t nv, int64_t n, int64_t grid_cap) {
    OccPart &q = it.p[it.np++];
    q.list = list;
    q.nv = nv;
    q.n = n;
    q.first_pt = it.pts;
    q.first_off = it.inc;
    if (n < 2 * nv) {                       // num_pts / num_voxels < 2.0, as an exact integer test
        q.per = 0;
        q.npts = n;
        it.inc += (uint64_t)(torch_uniform_inc(n, grid_cap) + torch_uniform_inc(3 * n, grid_cap));
    } else {
        q.per = n / nv + 1;
        q.npts = nv * q.per;
        it.inc += (uint64_t)torch_uniform_inc(3 * q.npts, grid_cap);
    }
    it.pts += q.npts;
}

__device__ __forceinline__ OccIter occ_iteration(bool warmup, const int64_t *__restrict__ counts, const int64_t *occupied, const int64_t *empty,
                                                 int64_t cells, int64_t num_pts, int64_t grid_cap) {
    OccIter it;
    it.np = 0;
    it.pts = 0;
    it.inc = 0;
    const int64_t n_occ = counts[0], n_empty = counts[1];
    it.empty_occupied = !warmup && n_occ == 0;
    if (it.empty_occupied) return it;
    if (warmup) {
        occ_add_part(it, nullptr, cells, num_pts, grid_cap);
    } else {
        occ_add_part(it, nullptr, cells, num_pts / 2, grid_cap);
        if (n_empty > 0) occ_add_part(it, empty, n_empty, num_pts / 4, grid_cap);
        occ_add_part(it, occupied, n_occ, num_pts / 4, grid_cap);
    }
    return it;
}

__global__ void __launch_bounds__(256)
k_occ_draw(const int64_t *__restrict__ rng, const int32_t *__restrict__ warmup, const int64_t *__restrict__ counts, const int64_t *occupied,
           const int64_t *empty, int rx, int ry, int rz, int num_steps, int64_t num_pts, int64_t grid_cap, float *__restrict__ pts,
           int64_t *__restrict__ out) {
    const int64_t cells = (int64_t)rx * ry * rz;
    const OccIter it = occ_iteration(*warmup != 0, counts, occupied, empty, cells, num_pts, grid_cap);
    const int64_t total = it.pts * num_steps;
    const uint64_t seed = (uint64_t)rng[0], base = (uint64_t)rng[1];
    const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i0 == 0) {
        out[0] = total;
        out[1] = it.empty_occupied ? 1 : 0;
    }
    const float res[3] = {(float)rx, (float)ry, (float)rz};
    for (int64_t i = i0; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = i / it.pts, r = i - s * it.pts;
        int k = 0;
        while (k + 1 < it.np && r >= it.p[k + 1].first_pt) ++k;
        const OccPart &q = it.p[k];
        const int64_t j = r - q.first_pt;
        const uint64_t off = base + (uint64_t)s * it.inc + q.first_off;
        int64_t v;
        float u[3];
        if (q.per == 0) {
            v = torch_randint_at(seed, off, j, torch_uniform_stride(q.n, grid_cap), (uint64_t)q.nv, 0);
            const uint64_t off_u = off + (uint64_t)torch_uniform_inc(q.n, grid_cap);
            const int64_t st = torch_uniform_stride(3 * q.n, grid_cap);
#pragma unroll
            for (int c = 0; c < 3; ++c) u[c] = torch_uniform_at(seed, off_u, 3 * j + c, st);
        } else {
            v = j / q.per;
            const int64_t st = torch_uniform_stride(3 * q.npts, grid_cap);
#pragma unroll
            for (int c = 0; c < 3; ++c) u[c] = torch_uniform_at(seed, off, 3 * j + c, st);
        }
        const int64_t cell = q.list ? q.list[v] : v;
        const int64_t g[3] = {cell / ((int64_t)ry * rz), (cell / rz) % ry, cell % rz};
#pragma unroll
        for (int c = 0; c < 3; ++c)       // ((gidx + off) / res) * 2 - 1, each op rounded as torch's elementwise kernels round it
            pts[3 * i + c] = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn((float)g[c], u[c]), res[c]), 2.f), 1.f);
    }
}

}  // namespace nsb

using namespace nsb;

extern "C" int nsb_occ_voxel_lists(const uint8_t *occ_grid, int64_t cells, int32_t *flags, int32_t *first, int64_t *occupied, int64_t *empty,
                                   int64_t *counts, void *workspace, void *stream) {
    NSB_REQUIRE(occ_grid && flags && first && occupied && empty && counts && workspace, "nsb_occ_voxel_lists: NULL argument");
    NSB_REQUIRE(cells > 0 && cells < ((int64_t)1 << 31), "nsb_occ_voxel_lists: the grid must hold 1 .. 2^31 - 1 cells (got %lld)", (long long)cells);
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaError_t e = cudaMemsetAsync(workspace, 0, (size_t)nsb_scan_workspace_bytes(), s)) {
        set_error("nsb_occ_voxel_lists: zeroing the scan workspace failed: %s", cudaGetErrorString(e));
        return 1;
    }
    k_occ_flags<<<wave_grid(cells, 256, 8), 256, 0, s>>>(occ_grid, cells, flags);
    if (int rc = check_launch("nsb_occ_voxel_lists(flags)")) return rc;
    // counts[0] (and [1], overwritten below) = the occupied cells; first = the occupied cells before each cell
    if (int rc = nsb_scan_counts(flags, cells, first, nullptr, occupied, nullptr, nullptr, nullptr, counts, nullptr, 0, workspace, stream)) return rc;
    k_occ_empty_list<<<wave_grid(cells, 256, 8), 256, 0, s>>>(flags, first, cells, empty, counts);
    return check_launch("nsb_occ_voxel_lists(empty)");
}

// the points one update may draw: per part at most max(n, nv (n // nv + 1)) <= n + min(nv, n / 2) (the second branch needs n >= 2 nv)
static int64_t occ_part_cap(int64_t n, int64_t cells) { return n + (cells < n / 2 ? cells : n / 2); }

// (fields/occ_update.py:capacity sizes the arena by the same bound)
static int64_t occ_draw_capacity(int64_t cells, int32_t num_steps, int64_t num_pts) {
    const int64_t warm = occ_part_cap(num_pts, cells);
    const int64_t steady = occ_part_cap(num_pts / 2, cells) + 2 * occ_part_cap(num_pts / 4, cells);
    return (int64_t)num_steps * (warm > steady ? warm : steady);
}

extern "C" int nsb_occ_draw_pts(const int64_t *rng, const int32_t *warmup, const int64_t *counts, const int64_t *occupied, const int64_t *empty,
                                int32_t rx, int32_t ry, int32_t rz, int32_t num_steps, int64_t num_pts, int64_t capacity, float *pts, int64_t *out,
                                void *stream) {
    NSB_REQUIRE(rng && warmup && counts && occupied && empty && pts && out, "nsb_occ_draw_pts: NULL argument");
    NSB_REQUIRE(rx > 0 && ry > 0 && rz > 0 && num_steps > 0 && num_pts >= 0, "nsb_occ_draw_pts: bad resolution, num_steps or num_pts");
    const int64_t cells = (int64_t)rx * ry * rz;
    NSB_REQUIRE(cells < ((int64_t)1 << 31), "nsb_occ_draw_pts: the grid must hold fewer than 2^31 cells");
    NSB_REQUIRE(3 * occ_part_cap(num_pts, cells) < ((int64_t)1 << 31),
                "nsb_occ_draw_pts: a draw of %lld points may reach 2^31 values, which torch splits into 32-bit sub-draws", (long long)num_pts);
    const int64_t need = occ_draw_capacity(cells, num_steps, num_pts);
    NSB_REQUIRE(capacity >= need, "nsb_occ_draw_pts: the point arena holds %lld points, an update may draw %lld", (long long)capacity, (long long)need);
    k_occ_draw<<<wave_grid(need, 256, 4), 256, 0, (cudaStream_t)stream>>>(rng, warmup, counts, occupied, empty, rx, ry, rz, num_steps, num_pts,
                                                                          torch_rand_grid_cap(), pts, out);
    return check_launch("nsb_occ_draw_pts");
}
