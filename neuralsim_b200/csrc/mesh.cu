// Marching cubes on a lattice streamed in slabs of whole planes along the first (slowest) axis -- the stages behind
// neuralsim_b200/graphics/trianglemesh.py:extract_mesh.
//
//   k_mc_lattice_points  the query points of a run of lattice points (x = (lin0[i], lin1[j], lin2[k]))
//   k_mc_count           per owned lattice point: crossing flags of the <= 3 edges it owns (+x, +y, +z) and their count;
//                        per cell (i - 1, j, k) of the same slot: case index and triangle count (mc_table.cuh)
//   k_mc_vertices        one vertex per set flag at slot first[l] + rank: position and interpolated lattice-gradient normal, in fp64
//   k_mc_triangles       the triangles of every cell at slot tfirst[l] + entry, with global vertex ids
//
// A slab owns lattice planes [p0, p1): their edges' vertices and the cells (p0 - 1 .. p1 - 2), i.e. the cells between the last plane of the
// previous slab (carried: its flags and scanned vertex offsets) and the owned planes.  The two count arrays go through nsb_scan_counts in
// between; nothing is placed by an atomic, so the output order is fixed by the scans and does not depend on the slab size.
#include "mc_table.cuh"
#include "nsb_common.cuh"

namespace nsb {

struct McGeom {
    int64_t n1, n2, plane;          // lattice dims 1, 2 and n1 n2
    int32_t n0, p0, p1, w0;         // dim 0, owned planes [p0, p1), first plane held by the sdf window
};

__device__ __forceinline__ float mc_s(const float *__restrict__ win, const McGeom &g, int64_t i, int64_t jk) {
    return win[(i - g.w0) * g.plane + jk];
}

__global__ void __launch_bounds__(256)
k_mc_lattice_points(const float *__restrict__ lin0, const float *__restrict__ lin1, const float *__restrict__ lin2, int64_t n1, int64_t n2,
                    int64_t start, int64_t n, float *__restrict__ x) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x, plane = n1 * n2;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += stride) {
        const int64_t f = start + q, i = f / plane, jk = f - i * plane, j = jk / n2, k = jk - j * n2;
        x[q * 3 + 0] = lin0[i];
        x[q * 3 + 1] = lin1[j];
        x[q * 3 + 2] = lin2[k];
    }
}

__global__ void __launch_bounds__(256)
k_mc_count(const float *__restrict__ win, McGeom g, double level, uint8_t *__restrict__ flags, int32_t *__restrict__ vcount,
           uint8_t *__restrict__ cases, int32_t *__restrict__ tcount) {
    const int64_t n = (int64_t)(g.p1 - g.p0) * g.plane, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n; l += stride) {
        const int64_t i = g.p0 + l / g.plane, jk = l % g.plane, j = jk / g.n2, k = jk - j * g.n2;
        const bool in0 = (double)mc_s(win, g, i, jk) < level;
        uint32_t f = 0;
        if (i + 1 < g.n0 && ((double)mc_s(win, g, i + 1, jk) < level) != in0) f |= 1u;
        if (j + 1 < g.n1 && ((double)mc_s(win, g, i, jk + g.n2) < level) != in0) f |= 2u;
        if (k + 1 < g.n2 && ((double)mc_s(win, g, i, jk + 1) < level) != in0) f |= 4u;
        flags[l] = (uint8_t)f;
        vcount[l] = __popc(f);
        uint32_t c = 0;
        if (i >= 1 && j + 1 < g.n1 && k + 1 < g.n2) {          // cell (i - 1, j, k): corner b at (i - 1 + (b & 1), j + (b >> 1 & 1), k + (b >> 2 & 1))
#pragma unroll
            for (int b = 0; b < 8; ++b)
                if ((double)mc_s(win, g, i - 1 + (b & 1), jk + (b >> 1 & 1) * g.n2 + (b >> 2 & 1)) < level) c |= 1u << b;
        }
        cases[l] = (uint8_t)c;
        tcount[l] = kMcTriCount[c];
    }
}

// d sdf / d axis at lattice point (i, j, k): central differences, one-sided at the volume border, over the spacing
__device__ __forceinline__ double mc_grad(const float *__restrict__ win, const McGeom &g, int64_t idx, int64_t dim, int64_t step,
                                          int64_t i, int64_t jk, double h) {
    const int64_t di = step == 0 ? 1 : 0, djk = step;          // step 0: axis 0 (plane index), else the jk stride of axis 1 / 2
    const double sp = idx + 1 < dim ? (double)mc_s(win, g, i + di, jk + djk) : (double)mc_s(win, g, i, jk);
    const double sm = idx > 0 ? (double)mc_s(win, g, i - di, jk - djk) : (double)mc_s(win, g, i, jk);
    return (idx > 0 && idx + 1 < dim) ? (sp - sm) / (2.0 * h) : (sp - sm) / h;
}

struct McVertArgs {
    double level, bmin[3], h[3];
};

// the vertex on the axis-A edge of lattice point (i, j, k) at slot `slot`; g0: the lattice gradient at (i, j, k)
template <int A>
__device__ __forceinline__ void mc_vertex(const float *__restrict__ win, const McGeom &g, const McVertArgs &v, int64_t i, int64_t j, int64_t k,
                                          int64_t jk, const double (&g0)[3], int64_t slot, float *__restrict__ verts, float *__restrict__ normals) {
    const int64_t i1 = A == 0 ? i + 1 : i, j1 = A == 1 ? j + 1 : j, k1 = A == 2 ? k + 1 : k, jk1 = jk + (A == 1 ? g.n2 : A == 2 ? 1 : 0);
    const double s0 = (double)mc_s(win, g, i, jk), s1 = (double)mc_s(win, g, i1, jk1);
    const double t = (v.level - s0) / (s1 - s0);
    const double g1[3] = {mc_grad(win, g, i1, g.n0, 0, i1, jk1, v.h[0]), mc_grad(win, g, j1, g.n1, g.n2, i1, jk1, v.h[1]),
                          mc_grad(win, g, k1, g.n2, 1, i1, jk1, v.h[2])};
    double nrm[3], nn = 0.0;
#pragma unroll
    for (int b = 0; b < 3; ++b) {
        nrm[b] = g0[b] + t * (g1[b] - g0[b]);
        nn += nrm[b] * nrm[b];
    }
    const double inv = nn > 0.0 ? 1.0 / sqrt(nn) : 0.0;
    const double idx[3] = {(double)i + (A == 0 ? t : 0.0), (double)j + (A == 1 ? t : 0.0), (double)k + (A == 2 ? t : 0.0)};
#pragma unroll
    for (int b = 0; b < 3; ++b) {
        verts[slot * 3 + b] = (float)(v.bmin[b] + v.h[b] * idx[b]);
        normals[slot * 3 + b] = (float)(nrm[b] * inv);
    }
}

// (256, 2): room for 128 registers -- the fp64 gradients of both edge ends spill at the default 64
__global__ void __launch_bounds__(256, 2)
k_mc_vertices(const float *__restrict__ win, McGeom g, McVertArgs v, const uint8_t *__restrict__ flags, const int32_t *__restrict__ vfirst,
              float *__restrict__ verts, float *__restrict__ normals) {
    const int64_t n = (int64_t)(g.p1 - g.p0) * g.plane, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n; l += stride) {
        const uint32_t f = flags[l];
        if (!f) continue;
        const int64_t i = g.p0 + l / g.plane, jk = l % g.plane, j = jk / g.n2, k = jk - j * g.n2;
        const double g0[3] = {mc_grad(win, g, i, g.n0, 0, i, jk, v.h[0]), mc_grad(win, g, j, g.n1, g.n2, i, jk, v.h[1]),
                              mc_grad(win, g, k, g.n2, 1, i, jk, v.h[2])};
        int64_t slot = vfirst[l];                                   // the point's vertices in axis order
        if (f & 1u) mc_vertex<0>(win, g, v, i, j, k, jk, g0, slot++, verts, normals);
        if (f & 2u) mc_vertex<1>(win, g, v, i, j, k, jk, g0, slot++, verts, normals);
        if (f & 4u) mc_vertex<2>(win, g, v, i, j, k, jk, g0, slot, verts, normals);
    }
}

__global__ void __launch_bounds__(256)
k_mc_triangles(McGeom g, const uint8_t *__restrict__ cases, const int32_t *__restrict__ tcount, const int32_t *__restrict__ tfirst,
               const uint8_t *__restrict__ flags, const int32_t *__restrict__ vfirst, int64_t vbase, const uint8_t *__restrict__ carry_flags,
               const int32_t *__restrict__ carry_first, int64_t carry_base, int32_t *__restrict__ faces) {
    const int64_t n = (int64_t)(g.p1 - g.p0) * g.plane, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n; l += stride) {
        const int cnt = tcount[l];
        if (!cnt) continue;
        const int c = cases[l];
        const int64_t ci = g.p0 - 1 + l / g.plane, jk = l % g.plane;      // cell (ci, j, k)
        const int64_t slot = tfirst[l];
        for (int q = 0; q < cnt * 3; ++q) {
            const int e = kMcTriEdges[c][q], a = e >> 2;
            const int64_t oi = ci + kMcEdgeOwner[e][0], ojk = jk + kMcEdgeOwner[e][1] * g.n2 + kMcEdgeOwner[e][2];
            const uint32_t below = (1u << a) - 1u;
            int64_t id;
            if (oi < g.p0) id = carry_base + carry_first[ojk] + __popc(carry_flags[ojk] & below);   // the plane carried from the previous slab
            else {
                const int64_t lo = (oi - g.p0) * g.plane + ojk;
                id = vbase + vfirst[lo] + __popc(flags[lo] & below);
            }
            faces[slot * 3 + q] = (int32_t)id;
        }
    }
}

}  // namespace nsb

using namespace nsb;
#define STREAM ((cudaStream_t)stream)

static int mc_geom(int32_t n0, int32_t n1, int32_t n2, int32_t p0, int32_t p1, int32_t w0, int32_t n_win, int32_t need_lo, int32_t need_hi,
                   const char *who, McGeom *g) {
    NSB_REQUIRE(n0 >= 2 && n1 >= 2 && n2 >= 2, "%s: lattice dims must be >= 2, got %d x %d x %d", who, n0, n1, n2);
    NSB_REQUIRE(0 <= p0 && p0 < p1 && p1 <= n0, "%s: owned planes [%d, %d) outside [0, %d)", who, p0, p1, n0);
    const int32_t lo = p0 - need_lo < 0 ? 0 : p0 - need_lo, hi = p1 + need_hi > n0 ? n0 : p1 + need_hi;
    NSB_REQUIRE(w0 <= lo && w0 + n_win >= hi, "%s: the sdf window [%d, %d) must hold planes [%d, %d)", who, w0, w0 + n_win, lo, hi);
    *g = McGeom{n1, n2, (int64_t)n1 * n2, n0, p0, p1, w0};
    return 0;
}

extern "C" int nsb_mc_lattice_points(const float *lin0, const float *lin1, const float *lin2, int32_t n1, int32_t n2, int64_t start,
                                     int64_t n, float *x, void *stream) {
    if (n == 0) return 0;
    NSB_REQUIRE(lin0 && lin1 && lin2 && x, "nsb_mc_lattice_points: NULL argument");
    k_mc_lattice_points<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(lin0, lin1, lin2, n1, n2, start, n, x);
    return check_launch("nsb_mc_lattice_points");
}

extern "C" int nsb_mc_count(const float *sdf_win, int32_t w0, int32_t n_win, int32_t n0, int32_t n1, int32_t n2, int32_t p0, int32_t p1,
                            double level, uint8_t *flags, int32_t *vcount, uint8_t *cases, int32_t *tcount, void *stream) {
    McGeom g;
    if (const int rc = mc_geom(n0, n1, n2, p0, p1, w0, n_win, 1, 1, "nsb_mc_count", &g)) return rc;
    NSB_REQUIRE(sdf_win && flags && vcount && cases && tcount, "nsb_mc_count: NULL argument");
    const int64_t n = (int64_t)(p1 - p0) * g.plane;
    k_mc_count<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(sdf_win, g, level, flags, vcount, cases, tcount);
    return check_launch("nsb_mc_count");
}

extern "C" int nsb_mc_vertices(const float *sdf_win, int32_t w0, int32_t n_win, int32_t n0, int32_t n1, int32_t n2, int32_t p0, int32_t p1,
                               double level, const double *bmin3_host, const double *spacing3_host, const uint8_t *flags, const int32_t *vfirst,
                               float *verts, float *normals, void *stream) {
    McGeom g;
    if (const int rc = mc_geom(n0, n1, n2, p0, p1, w0, n_win, 1, 2, "nsb_mc_vertices", &g)) return rc;
    NSB_REQUIRE(sdf_win && bmin3_host && spacing3_host && flags && vfirst && verts && normals, "nsb_mc_vertices: NULL argument");
    const int64_t n = (int64_t)(p1 - p0) * g.plane;
    McVertArgs v{level, {bmin3_host[0], bmin3_host[1], bmin3_host[2]}, {spacing3_host[0], spacing3_host[1], spacing3_host[2]}};
    k_mc_vertices<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(sdf_win, g, v, flags, vfirst, verts, normals);
    return check_launch("nsb_mc_vertices");
}

extern "C" int nsb_mc_triangles(int32_t n0, int32_t n1, int32_t n2, int32_t p0, int32_t p1, const uint8_t *cases, const int32_t *tcount,
                                const int32_t *tfirst, const uint8_t *flags, const int32_t *vfirst, int64_t vbase, const uint8_t *carry_flags,
                                const int32_t *carry_first, int64_t carry_base, int32_t *faces, void *stream) {
    McGeom g;
    if (const int rc = mc_geom(n0, n1, n2, p0, p1, 0, n0, 0, 0, "nsb_mc_triangles", &g)) return rc;
    NSB_REQUIRE(cases && tcount && tfirst && flags && vfirst && faces, "nsb_mc_triangles: NULL argument");
    NSB_REQUIRE(p0 == 0 || (carry_flags && carry_first), "nsb_mc_triangles: a slab after the first needs the carried plane");
    const int64_t n = (int64_t)(p1 - p0) * g.plane;
    k_mc_triangles<<<wave_grid(n, 256, 8), 256, 0, STREAM>>>(g, cases, tcount, tfirst, flags, vfirst, vbase, carry_flags, carry_first,
                                                              carry_base, faces);
    return check_launch("nsb_mc_triangles");
}
