// nnps_kernels.cuh -- cell keys, counting sort, cell-relative repack, neighbour query.
// Part of the single translation unit b200sph.cu (included there, in this order; not a
// stand-alone header).

// --------------------------------------------------------------------------
// NNPS build kernels
// --------------------------------------------------------------------------

// cell id = floor((p - xmin)/cell) per axis (find_cell_id_raw, nnps_base.pxd:39-80),
// flat = cx + ncx*cy + ncx*ncy*cz (flatten_raw, nnps_base.pxd:84-96) or, zorder, cx + ncx *
// morton(cy, cz) (z_order.h:24-46 interleaves all three; see grid_row); the arrival
// counter replaces the linked-list push (linked_list_nnps.pyx:285-286).
__global__ void k_cell_count(const double *__restrict__ x, const double *__restrict__ y,
                             const double *__restrict__ z, const uint8_t *__restrict__ ptype,
                             long long pool_end, GridDev G, uint32_t *__restrict__ key_of,
                             uint32_t *__restrict__ off_in, uint32_t *__restrict__ cell_cnt)
{
    long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= pool_end) return;
    if (ptype[g] == PT_INVALID) return;
    int cx = (int)floor((x[g] - G.xmin[0]) / G.cell[0]);
    int cy = (int)floor((y[g] - G.xmin[1]) / G.cell[1]);
    int cz = (int)floor((z[g] - G.xmin[2]) / G.cell[2]);
    cx = min(max(cx, 0), G.nc[0] - 1);
    cy = min(max(cy, 0), G.nc[1] - 1);
    cz = min(max(cz, 0), G.nc[2] - 1);
    uint32_t key = (uint32_t)cx + (uint32_t)G.nc[0] * grid_row(G.zorder, (uint32_t)G.nc[1], (uint32_t)cy, (uint32_t)cz);
    key_of[g] = key;
    off_in[g] = atomicAdd(&cell_cnt[key], 1u);
}

__global__ void k_scatter(const uint32_t *__restrict__ key_of, const uint32_t *__restrict__ off_in,
                          const uint8_t *__restrict__ ptype, long long pool_end,
                          const uint32_t *__restrict__ cell_start, uint32_t *__restrict__ perm_tmp)
{
    long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= pool_end) return;
    if (ptype[g] == PT_INVALID) return;
    perm_tmp[cell_start[key_of[g]] + off_in[g]] = (uint32_t)g;
}

// make the order inside every cell canonical (ascending pool index) so that the
// build -- and therefore every fp32 sum downstream -- is run-to-run deterministic.
__global__ void k_canon(const uint32_t *__restrict__ perm_tmp, const uint32_t *__restrict__ key_of,
                        const uint32_t *__restrict__ cell_start, long long n,
                        uint32_t *__restrict__ perm, uint32_t *__restrict__ skey,
                        uint32_t *__restrict__ rank)
{
    long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t g = perm_tmp[s];
    const uint32_t key = key_of[g];
    const uint32_t cs = cell_start[key], ce = cell_start[key + 1];
    uint32_t r = 0;
    for (uint32_t t = cs; t < ce; t++) r += (perm_tmp[t] < g) ? 1u : 0u;
    const uint32_t d = cs + r;
    perm[d] = g;
    skey[d] = key;
    rank[g] = d;
}

// A[s] = (x, y, z relative to the particle's own cell origin, h)
__global__ void k_pack_pos(const double *__restrict__ x, const double *__restrict__ y,
                           const double *__restrict__ z, const double *__restrict__ h,
                           const uint32_t *__restrict__ perm, const uint32_t *__restrict__ skey,
                           long long n, GridDev G, float4 *__restrict__ A, float4 *__restrict__ AB,
                           const uint8_t *__restrict__ ptype, uint8_t *__restrict__ stype)
{
    long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t g = perm[s];
    if (stype) stype[s] = ptype[g];
    const float4 a = pack_position(G, skey[s], x[g], y[g], z[g], h[g]);
    A[s] = a;
    AB[2 * s] = a;
}

// refresh the packed positions in the FROZEN sorted order / cell frames of the last
// build and measure how far particles moved (and h grew) since then.
// red_u32[0] = max |dx|^2 (float bits), red_u32[1] = max (h - h_build) (float bits, >= 0)
__global__ void k_pack_pos_light(const double *__restrict__ x, const double *__restrict__ y,
                                 const double *__restrict__ z, const double *__restrict__ h,
                                 const uint32_t *__restrict__ perm, const uint32_t *__restrict__ skey,
                                 long long n, GridDev G, const float4 *__restrict__ A0,
                                 float4 *__restrict__ A, float4 *__restrict__ AB,
                                 unsigned *__restrict__ red_u32)
{
    long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float d2 = 0.f, dh = 0.f;
    if (s < n) {
        const uint32_t g = perm[s];
        const float4 a = pack_position(G, skey[s], x[g], y[g], z[g], h[g]);
        A[s] = a;
        AB[2 * s] = a;
        build_drift(a, A0[s], d2, dh);
    }
    for (int o = 16; o > 0; o >>= 1) {
        d2 = fmaxf(d2, __shfl_xor_sync(0xffffffffu, d2, o));
        dh = fmaxf(dh, __shfl_xor_sync(0xffffffffu, dh, o));
    }
    if ((threadIdx.x & 31) == 0) {
        if (d2 > 0.f) atomicMax(&red_u32[0], __float_as_uint(d2));
        if (dh > 0.f) atomicMax(&red_u32[1], __float_as_uint(dh));
    }
}

// B[s] = (u, v, w, m);  C[s] = (rho, p/rho^2, cs, type); pending TaitEOS /
// TaitEOSHGCorrection calls (wc/basic.py:60-65,118-126) are applied on the way
__global__ void k_pack_state(const double *__restrict__ u, const double *__restrict__ v,
                             const double *__restrict__ w, const double *__restrict__ m,
                             double *__restrict__ rho, float *__restrict__ p,
                             float *__restrict__ cs, const uint8_t *__restrict__ ptype,
                             const uint32_t *__restrict__ perm, long long n,
                             float4 *__restrict__ B, float4 *__restrict__ C,
                             float4 *__restrict__ AB, const EosTab E, const int eos_any)
{
    long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t g = perm[s];
    const int t = (int)ptype[g];
    double r = rho[g];
    float pg, csg;
    if (eos_any && eos_tab_applies(E, (uint8_t)t)) {
        if (eos_tab_eval(E, t & 7, r, pg, csg)) rho[g] = r;
        p[g] = pg;
        cs[g] = csg;
    } else {
        pg = p[g];
        csg = cs[g];
    }
    float4 b, c;
    state_record(u[g], v[g], w[g], m[g], r, pg, csg, t, b, c);
    B[s] = b;
    C[s] = c;
    AB[2 * s + 1] = b;
}

// neighbour query for one destination particle with the pair kernel's accept test
// (cell by cell; periodic axes wrap).  One warp.
__global__ void k_neighbors(const float4 *__restrict__ A /* {A,B} interleaved: A of particle s at [2 s] */, const float4 *__restrict__ C,
                            const uint32_t *__restrict__ cell_start, const uint32_t *__restrict__ skey,
                            const uint32_t *__restrict__ perm, long long s, int src_arr,
                            long long src_off, GridDev G, float k2,
                            uint32_t *__restrict__ out, long long cap, unsigned long long *count)
{
    const int lane = threadIdx.x;
    const int ncx = G.nc[0], ncy = G.nc[1], ncz = G.nc[2];
    const float4 Ai = A[2 * (size_t)s];
    uint32_t kq = skey[s];
    uint32_t ucx, ucy, ucz;
    grid_decode(G.zorder, (uint32_t)ncx, (uint32_t)ncy, kq, ucx, ucy, ucz);
    const int cx = (int)ucx, cy = (int)ucy, cz = (int)ucz;
    const float hi2 = k2 * Ai.w * Ai.w;
    unsigned long long n = 0;
    for (int r = 0; r < 27; r++) {
        const int dx = (r % 3) - 1, dy = ((r / 3) % 3) - 1, dz = (r / 9) - 1;
        int xx = cx + dx, yy = cy + dy, zz = cz + dz;
        if (G.periodic[0]) xx = (xx + ncx) % ncx;
        if (G.periodic[1]) yy = (yy + ncy) % ncy;
        if (G.periodic[2]) zz = (zz + ncz) % ncz;
        if (xx < 0 || xx >= ncx || yy < 0 || yy >= ncy || zz < 0 || zz >= ncz) continue;
        const uint32_t c = (uint32_t)xx + (uint32_t)ncx * grid_row(G.zorder, (uint32_t)ncy, (uint32_t)yy, (uint32_t)zz);
        const uint32_t rs = cell_start[c], re = cell_start[c + 1];
        for (uint32_t t0 = rs; t0 < re; t0 += 32) {
            const uint32_t t = t0 + lane;
            bool ok = false;
            if (t < re) {
                const float4 Aj = A[2 * (size_t)t];
                const float xij = Ai.x - (float)dx * (float)G.cell[0] - Aj.x;
                const float yij = Ai.y - (float)dy * (float)G.cell[1] - Aj.y;
                const float zij = Ai.z - (float)dz * (float)G.cell[2] - Aj.z;
                const float r2 = xij * xij + yij * yij + zij * zij;
                ok = ((r2 < hi2) || (r2 < k2 * Aj.w * Aj.w)) &&
                     ((__float_as_int(C[t].w) & 7) == src_arr);
            }
            const unsigned m = __ballot_sync(0xffffffffu, ok);
            if (ok) {
                const unsigned long long pos = n + __popc(m & ((1u << lane) - 1u));
                if ((long long)pos < cap) out[pos] = (uint32_t)((long long)perm[t] - src_off);
            }
            n += __popc(m);
        }
    }
    if (lane == 0) *count = n;
}
