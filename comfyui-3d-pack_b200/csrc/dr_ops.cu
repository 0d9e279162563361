// Mesh attribute ops on the rasterizer output: interpolate, bilinear texture, silhouette antialias
// (+ backward passes) and the edge-topology build used by antialias.
//
// Replace nvdiffrast's dr.interpolate / dr.texture(filter_mode='linear') / dr.antialias for the reference's
// call sites (diff_mesh_renderer.py:101-138, flexicubes_renderer.py:55-66, FlexiCubes/util.py:90-93,
// mesh_utils.py:534).  All four are one-pass, per-pixel, HBM/L2-bound kernels: full-frame buffers are read
// once with 128-bit accesses where the layout allows, vertex attributes / texels are gathered through L2,
// gradients to shared data (attributes, texels, vertex positions) leave as red.global.add.
#include "../../include/dr_b200.h"
#include "gs_common.cuh"

namespace {

// ------------------------------------------------------------------------------------------- interpolate
__global__ void __launch_bounds__(256)
interpolate_fwd_kernel(const float* __restrict__ attr, int attr_B, const float4* __restrict__ rast,
                       const int32_t* __restrict__ tri, const float4* __restrict__ rast_db, int B, int V, int H, int W,
                       int A, float* __restrict__ out, float* __restrict__ out_da) {
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t npix = (size_t)B * H * W;
    if (pix >= npix) return;
    const float4 r = rast[pix];
    const int f = (int)r.w - 1;
    float* o = out + pix * A;
    float* oda = out_da ? out_da + pix * 2 * A : nullptr;
    if (f < 0) {
        for (int a = 0; a < A; a++) o[a] = 0.f;
        if (oda) for (int a = 0; a < 2 * A; a++) oda[a] = 0.f;
        return;
    }
    const int b = (int)(pix / ((size_t)H * W));
    const float* ab = attr + (attr_B > 1 ? (size_t)b * V * A : 0);
    const float* a0 = ab + (size_t)tri[3 * f] * A;
    const float* a1 = ab + (size_t)tri[3 * f + 1] * A;
    const float* a2 = ab + (size_t)tri[3 * f + 2] * A;
    const float u = r.x, v = r.y, w2 = 1.0f - r.x - r.y;
    float4 db = make_float4(0.f, 0.f, 0.f, 0.f);
    if (oda) db = rast_db[pix];
    for (int a = 0; a < A; a++) {
        const float x0 = __ldg(a0 + a), x1 = __ldg(a1 + a), x2 = __ldg(a2 + a);
        o[a] = u * x0 + v * x1 + w2 * x2;
        if (oda) {
            const float d0 = x0 - x2, d1 = x1 - x2;
            oda[2 * a] = db.x * d0 + db.z * d1;
            oda[2 * a + 1] = db.y * d0 + db.w * d1;
        }
    }
}

__global__ void __launch_bounds__(256)
interpolate_bwd_kernel(const float* __restrict__ attr, int attr_B, const float4* __restrict__ rast,
                       const int32_t* __restrict__ tri, const float4* __restrict__ rast_db, int B, int V, int H, int W,
                       int A, const float* __restrict__ g_out, const float* __restrict__ g_da,
                       float* __restrict__ d_attr, float4* __restrict__ d_rast, float4* __restrict__ d_db) {
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t npix = (size_t)B * H * W;
    if (pix >= npix) return;
    const float4 r = rast[pix];
    const int f = (int)r.w - 1;
    float4 gr = make_float4(0.f, 0.f, 0.f, 0.f), gdb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (f >= 0) {
        const int b = (int)(pix / ((size_t)H * W));
        const size_t boff = attr_B > 1 ? (size_t)b * V * A : 0;
        const int i0 = tri[3 * f], i1 = tri[3 * f + 1], i2 = tri[3 * f + 2];
        const float* a0 = attr + boff + (size_t)i0 * A;
        const float* a1 = attr + boff + (size_t)i1 * A;
        const float* a2 = attr + boff + (size_t)i2 * A;
        float* g0 = d_attr + boff + (size_t)i0 * A;
        float* g1 = d_attr + boff + (size_t)i1 * A;
        float* g2 = d_attr + boff + (size_t)i2 * A;
        const float u = r.x, v = r.y, w2 = 1.0f - r.x - r.y;
        float4 db = make_float4(0.f, 0.f, 0.f, 0.f);
        if (g_da) db = rast_db[pix];
        for (int a = 0; a < A; a++) {
            const float go = g_out[pix * A + a];
            const float d0 = __ldg(a0 + a) - __ldg(a2 + a), d1 = __ldg(a1 + a) - __ldg(a2 + a);
            gr.x += go * d0; gr.y += go * d1;
            float t0 = u * go, t1 = v * go, t2 = w2 * go;
            if (g_da) {
                const float gx = g_da[pix * 2 * A + 2 * a], gy = g_da[pix * 2 * A + 2 * a + 1];
                gdb.x += gx * d0; gdb.z += gx * d1; gdb.y += gy * d0; gdb.w += gy * d1;
                const float c0 = db.x * gx + db.y * gy, c1 = db.z * gx + db.w * gy;     // d(da)/d(a0 - a2), d(a1 - a2)
                t0 += c0; t1 += c1; t2 -= c0 + c1;
            }
            if (t0 != 0.f) atomicAdd(g0 + a, t0);
            if (t1 != 0.f) atomicAdd(g1 + a, t1);
            if (t2 != 0.f) atomicAdd(g2 + a, t2);
        }
    }
    d_rast[pix] = gr;
    if (d_db) d_db[pix] = gdb;
}

// ------------------------------------------------------------------------------------------- texture
__device__ __forceinline__ int wrap_or_clamp(int i, int n, int boundary) {
    if (boundary == 0) { i %= n; return i < 0 ? i + n : i; }
    return min(max(i, 0), n - 1);
}

__global__ void __launch_bounds__(256)
texture_fwd_kernel(const float* __restrict__ tex, int tex_B, int Ht, int Wt, int C, const float2* __restrict__ uv,
                   int B, int H, int W, int boundary, float* __restrict__ out) {
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t npix = (size_t)B * H * W;
    if (pix >= npix) return;
    const float2 t = uv[pix];
    const float x = t.x * Wt - 0.5f, y = t.y * Ht - 0.5f;
    const float xf = floorf(x), yf = floorf(y);
    const float fx = x - xf, fy = y - yf;
    const int x0 = wrap_or_clamp((int)xf, Wt, boundary), x1 = wrap_or_clamp((int)xf + 1, Wt, boundary);
    const int y0 = wrap_or_clamp((int)yf, Ht, boundary), y1 = wrap_or_clamp((int)yf + 1, Ht, boundary);
    const int b = (int)(pix / ((size_t)H * W));
    const float* tb = tex + (tex_B > 1 ? (size_t)b * Ht * Wt * C : 0);
    const float* t00 = tb + ((size_t)y0 * Wt + x0) * C; const float* t10 = tb + ((size_t)y0 * Wt + x1) * C;
    const float* t01 = tb + ((size_t)y1 * Wt + x0) * C; const float* t11 = tb + ((size_t)y1 * Wt + x1) * C;
    for (int c = 0; c < C; c++) {
        const float top = __ldg(t00 + c) * (1.f - fx) + __ldg(t10 + c) * fx;
        const float bot = __ldg(t01 + c) * (1.f - fx) + __ldg(t11 + c) * fx;
        out[pix * C + c] = top * (1.f - fy) + bot * fy;
    }
}

__global__ void __launch_bounds__(256)
texture_bwd_kernel(const float* __restrict__ tex, int tex_B, int Ht, int Wt, int C, const float2* __restrict__ uv,
                   int B, int H, int W, int boundary, const float* __restrict__ g_out, float* __restrict__ d_tex,
                   float2* __restrict__ d_uv) {
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t npix = (size_t)B * H * W;
    if (pix >= npix) return;
    const float2 t = uv[pix];
    const float x = t.x * Wt - 0.5f, y = t.y * Ht - 0.5f;
    const float xf = floorf(x), yf = floorf(y);
    const float fx = x - xf, fy = y - yf;
    const int x0 = wrap_or_clamp((int)xf, Wt, boundary), x1 = wrap_or_clamp((int)xf + 1, Wt, boundary);
    const int y0 = wrap_or_clamp((int)yf, Ht, boundary), y1 = wrap_or_clamp((int)yf + 1, Ht, boundary);
    const int b = (int)(pix / ((size_t)H * W));
    const size_t boff = tex_B > 1 ? (size_t)b * Ht * Wt * C : 0;
    const size_t o00 = boff + ((size_t)y0 * Wt + x0) * C, o10 = boff + ((size_t)y0 * Wt + x1) * C;
    const size_t o01 = boff + ((size_t)y1 * Wt + x0) * C, o11 = boff + ((size_t)y1 * Wt + x1) * C;
    float gx = 0.f, gy = 0.f;
    for (int c = 0; c < C; c++) {
        const float g = g_out[pix * C + c];
        if (g == 0.f) continue;
        const float v00 = __ldg(tex + o00 + c), v10 = __ldg(tex + o10 + c), v01 = __ldg(tex + o01 + c), v11 = __ldg(tex + o11 + c);
        gx += g * ((v10 - v00) * (1.f - fy) + (v11 - v01) * fy);
        gy += g * ((v01 * (1.f - fx) + v11 * fx) - (v00 * (1.f - fx) + v10 * fx));
        atomicAdd(d_tex + o00 + c, g * (1.f - fx) * (1.f - fy));
        atomicAdd(d_tex + o10 + c, g * fx * (1.f - fy));
        atomicAdd(d_tex + o01 + c, g * (1.f - fx) * fy);
        atomicAdd(d_tex + o11 + c, g * fx * fy);
    }
    d_uv[pix] = make_float2(gx * Wt, gy * Ht);
}

// ------------------------------------------------------------------------------------------- topology
__global__ void __launch_bounds__(256)
topo_emit_kernel(const int32_t* __restrict__ tri, int F, uint32_t* __restrict__ key_hi, uint32_t* __restrict__ idx) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;       // edge index = f*3 + e ; edge e joins vertices e+1, e+2
    if (i >= 3 * F) return;
    const int f = i / 3, e = i - 3 * f;
    const int va = tri[3 * f + (e + 1) % 3], vb = tri[3 * f + (e + 2) % 3];
    key_hi[i] = (uint32_t)max(va, vb);
    idx[i] = (uint32_t)i;
}
__global__ void __launch_bounds__(256)
topo_lo_kernel(const int32_t* __restrict__ tri, int F, const uint32_t* __restrict__ idx, uint32_t* __restrict__ key_lo) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * F) return;
    const int j = (int)idx[i], f = j / 3, e = j - 3 * f;
    key_lo[i] = (uint32_t)min(tri[3 * f + (e + 1) % 3], tri[3 * f + (e + 2) % 3]);
}
__device__ __forceinline__ uint2 edge_key(const int32_t* tri, int j) {
    const int f = j / 3, e = j - 3 * f;
    const int va = tri[3 * f + (e + 1) % 3], vb = tri[3 * f + (e + 2) % 3];
    return make_uint2((uint32_t)min(va, vb), (uint32_t)max(va, vb));
}
__global__ void __launch_bounds__(256)
topo_pair_kernel(const int32_t* __restrict__ tri, int F, const uint32_t* __restrict__ idx, int32_t* __restrict__ opp) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = 3 * F;
    if (i >= n) return;
    const int j = (int)idx[i];
    const uint2 k = edge_key(tri, j);
    int partner = -1;
    if (i > 0) { const int jp = (int)idx[i - 1]; const uint2 kp = edge_key(tri, jp); if (kp.x == k.x && kp.y == k.y) partner = jp; }
    if (partner < 0 && i + 1 < n) { const int jn = (int)idx[i + 1]; const uint2 kn = edge_key(tri, jn); if (kn.x == k.x && kn.y == k.y) partner = jn; }
    opp[j] = partner >= 0 ? tri[partner] : -1;           // tri[f*3+e] = vertex opposite edge e of triangle f
}

// ------------------------------------------------------------------------------------------- antialias
struct AAResult { bool found; bool to_b; float t; int tsel; int e; int ax, ay, bx, by; float dir; };

// Analysis of one adjacent pixel pair (x,y)-(x+1,y) [d=0] or (x,y)-(x,y+1) [d=1]; same decisions in fwd and bwd.
__device__ __forceinline__ AAResult aa_analyse(const float4* __restrict__ rast, const float4* __restrict__ pos,
                                               const int32_t* __restrict__ tri, const int32_t* __restrict__ opp, int b,
                                               int V, int H, int W, int x, int y, int d) {
    AAResult R; R.found = false;
    const size_t base = (size_t)b * H * W;
    const int x1 = x + (d == 0), y1 = y + (d == 1);
    const float4 r0 = rast[base + (size_t)y * W + x], r1 = rast[base + (size_t)y1 * W + x1];
    const int i0 = (int)r0.w, i1 = (int)r1.w;
    if (i0 == i1) return R;
    const bool use0 = (i1 == 0) || ((i0 > 0) && (r0.z < r1.z));
    R.tsel = (use0 ? i0 : i1) - 1;
    R.ax = use0 ? x : x1; R.ay = use0 ? y : y1; R.bx = use0 ? x1 : x; R.by = use0 ? y1 : y;
    const float cax = R.ax + 0.5f, cay = R.ay + 0.5f;
    R.dir = (d == 0) ? (float)(R.bx - R.ax) : (float)(R.by - R.ay);
    const int vi[3] = {tri[3 * R.tsel], tri[3 * R.tsel + 1], tri[3 * R.tsel + 2]};
    float2 S[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float4 p = pos[(size_t)b * V + vi[k]];
        if (!(p.w > 0.f)) return R;
        S[k] = make_float2((p.x / p.w + 1.0f) * (0.5f * W), (p.y / p.w + 1.0f) * (0.5f * H));
    }
#pragma unroll
    for (int e = 0; e < 3; e++) {
        const float2 Pa = S[(e + 1) % 3], Pb = S[(e + 2) % 3], Pc = S[e];
        const int op = opp[3 * R.tsel + e];
        bool sil = op < 0;
        if (!sil) {
            const float4 po = pos[(size_t)b * V + op];
            if (po.w > 0.f) {
                const float2 Po = make_float2((po.x / po.w + 1.0f) * (0.5f * W), (po.y / po.w + 1.0f) * (0.5f * H));
                const float ex = Pb.x - Pa.x, ey = Pb.y - Pa.y;
                const float sc = ex * (Pc.y - Pa.y) - ey * (Pc.x - Pa.x);
                const float so = ex * (Po.y - Pa.y) - ey * (Po.x - Pa.x);
                sil = sc * so > 0.f;
            }
        }
        if (!sil) continue;
        const float fa = (d == 0) ? Pa.y - cay : Pa.x - cax, fb = (d == 0) ? Pb.y - cay : Pb.x - cax;
        if (!(((fa <= 0.f) && (fb > 0.f)) || ((fb <= 0.f) && (fa > 0.f)))) continue;
        const float sp = -fa / (fb - fa);
        const float pa = (d == 0) ? Pa.x : Pa.y, pb = (d == 0) ? Pb.x : Pb.y, ca = (d == 0) ? cax : cay;
        const float cross = pa + sp * (pb - pa);
        const float t = (cross - ca) / R.dir;
        if (!(t >= 0.f && t <= 1.f)) continue;
        R.found = true; R.t = t; R.e = e; R.to_b = t > 0.5f;
        return R;
    }
    return R;
}

__global__ void __launch_bounds__(256)
antialias_fwd_kernel(const float* __restrict__ color, const float4* __restrict__ rast, const float4* __restrict__ pos,
                     const int32_t* __restrict__ tri, const int32_t* __restrict__ opp, int B, int V, int H, int W, int C,
                     float* __restrict__ out) {
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t npix = (size_t)B * H * W;
    if (pix >= npix) return;
    const int b = (int)(pix / ((size_t)H * W));
    const int rem = (int)(pix - (size_t)b * H * W);
    const int y = rem / W, x = rem - y * W;
    for (int d = 0; d < 2; d++) {
        if ((d == 0 && x + 1 >= W) || (d == 1 && y + 1 >= H)) continue;
        const AAResult R = aa_analyse(rast, pos, tri, opp, b, V, H, W, x, y, d);
        if (!R.found) continue;
        const size_t pa = ((size_t)b * H * W + (size_t)R.ay * W + R.ax) * C, pb = ((size_t)b * H * W + (size_t)R.by * W + R.bx) * C;
        const float wgt = R.to_b ? R.t - 0.5f : 0.5f - R.t;
        const size_t dst = R.to_b ? pb : pa;
        for (int c = 0; c < C; c++) {
            const float ca = color[pa + c], cb = color[pb + c];
            atomicAdd(out + dst + c, R.to_b ? wgt * (ca - cb) : wgt * (cb - ca));
        }
    }
}

__global__ void __launch_bounds__(256)
antialias_bwd_kernel(const float* __restrict__ color, const float4* __restrict__ rast, const float4* __restrict__ pos,
                     const int32_t* __restrict__ tri, const int32_t* __restrict__ opp, int B, int V, int H, int W, int C,
                     const float* __restrict__ g_out, float* __restrict__ d_color, float* __restrict__ d_pos) {
    const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t npix = (size_t)B * H * W;
    if (pix >= npix) return;
    const int b = (int)(pix / ((size_t)H * W));
    const int rem = (int)(pix - (size_t)b * H * W);
    const int y = rem / W, x = rem - y * W;
    for (int d = 0; d < 2; d++) {
        if ((d == 0 && x + 1 >= W) || (d == 1 && y + 1 >= H)) continue;
        const AAResult R = aa_analyse(rast, pos, tri, opp, b, V, H, W, x, y, d);
        if (!R.found) continue;
        const size_t pa = ((size_t)b * H * W + (size_t)R.ay * W + R.ax) * C, pb = ((size_t)b * H * W + (size_t)R.by * W + R.bx) * C;
        const float wgt = R.to_b ? R.t - 0.5f : 0.5f - R.t;
        const size_t dst = R.to_b ? pb : pa;
        float dt = 0.f;
        for (int c = 0; c < C; c++) {
            const float g = g_out[dst + c];
            const float ca = color[pa + c], cb = color[pb + c];
            // out[dst] += to_b ? (t-.5)(ca-cb) : (.5-t)(cb-ca)   -> both have d/dt = (ca - cb)
            dt += g * (ca - cb);
            const float gw = g * wgt;
            atomicAdd(d_color + pa + c, R.to_b ? gw : -gw);
            atomicAdd(d_color + pb + c, R.to_b ? -gw : gw);
        }
        if (dt == 0.f) continue;
        // t = (cross - cA)/dir, cross = pa + sp (pb - pa), sp = -fa/(fb - fa)
        const int va = tri[3 * R.tsel + (R.e + 1) % 3], vb = tri[3 * R.tsel + (R.e + 2) % 3];
        const float4 A4 = pos[(size_t)b * V + va], B4 = pos[(size_t)b * V + vb];
        const float2 Pa = make_float2((A4.x / A4.w + 1.0f) * (0.5f * W), (A4.y / A4.w + 1.0f) * (0.5f * H));
        const float2 Pb = make_float2((B4.x / B4.w + 1.0f) * (0.5f * W), (B4.y / B4.w + 1.0f) * (0.5f * H));
        const float cax = R.ax + 0.5f, cay = R.ay + 0.5f;
        const float fa = (d == 0) ? Pa.y - cay : Pa.x - cax, fb = (d == 0) ? Pb.y - cay : Pb.x - cax;
        const float den = fb - fa, sp = -fa / den;
        const float pa_ = (d == 0) ? Pa.x : Pa.y, pb_ = (d == 0) ? Pb.x : Pb.y;
        const float dcross = dt / R.dir;
        const float g_pa_ax = dcross * (1.f - sp), g_pb_ax = dcross * sp;
        const float g_sp = dcross * (pb_ - pa_);
        const float g_fa = g_sp * (-fb / (den * den)), g_fb = g_sp * (fa / (den * den));
        // screen-space gradients of the two edge endpoints: (ax = crossing axis, fix = the other one)
        const float gPa_x = (d == 0) ? g_pa_ax : g_fa, gPa_y = (d == 0) ? g_fa : g_pa_ax;
        const float gPb_x = (d == 0) ? g_pb_ax : g_fb, gPb_y = (d == 0) ? g_fb : g_pb_ax;
        // screen -> clip: Px = (x/w + 1) W/2
        float* da = d_pos + ((size_t)b * V + va) * 4;
        float* db = d_pos + ((size_t)b * V + vb) * 4;
        const float hw = 0.5f * W, hh = 0.5f * H;
        atomicAdd(da + 0, gPa_x * hw / A4.w); atomicAdd(da + 1, gPa_y * hh / A4.w);
        atomicAdd(da + 3, -(gPa_x * hw * A4.x + gPa_y * hh * A4.y) / (A4.w * A4.w));
        atomicAdd(db + 0, gPb_x * hw / B4.w); atomicAdd(db + 1, gPb_y * hh / B4.w);
        atomicAdd(db + 3, -(gPb_x * hw * B4.x + gPb_y * hh * B4.y) / (B4.w * B4.w));
    }
}

}  // namespace

#define DR_GRID(n) (unsigned)(((n) + 255) / 256), 256

extern "C" {

int32_t dr_b200_interpolate_fwd(const float* attr, int32_t attr_B, const float* rast, const int32_t* tri, const float* rast_db,
                                int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t A, float* out, float* out_da,
                                void* stream) {
    GS_REQ(attr && rast && tri && out, "NULL pointer");
    GS_REQ(attr_B == 1 || attr_B == B, "attr batch must be 1 or B");
    GS_REQ((out_da == nullptr) || (rast_db != nullptr), "out_da needs rast_db");
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t npix = (size_t)B * H * W;
    if (npix == 0) return 0;
    interpolate_fwd_kernel<<<DR_GRID(npix), 0, s>>>(attr, attr_B, (const float4*)rast, tri, (const float4*)rast_db, B, V, H, W, A, out, out_da);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int32_t dr_b200_interpolate_bwd(const float* attr, int32_t attr_B, const float* rast, const int32_t* tri, const float* rast_db,
                                int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t A, const float* g_out,
                                const float* g_da, float* d_attr, float* d_rast, float* d_db, void* stream) {
    GS_REQ(attr && rast && tri && g_out && d_attr && d_rast, "NULL pointer");
    GS_REQ((g_da == nullptr) || (rast_db != nullptr), "dL_dout_da needs rast_db");
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t npix = (size_t)B * H * W;
    if (npix == 0) return 0;
    interpolate_bwd_kernel<<<DR_GRID(npix), 0, s>>>(attr, attr_B, (const float4*)rast, tri, (const float4*)rast_db, B, V, H, W, A,
                                                    g_out, g_da, d_attr, (float4*)d_rast, (float4*)d_db);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int32_t dr_b200_texture_fwd(const float* tex, int32_t tex_B, int32_t Ht, int32_t Wt, int32_t C, const float* uv, int32_t B,
                            int32_t H, int32_t W, int32_t boundary, float* out, void* stream) {
    GS_REQ(tex && uv && out && Ht > 0 && Wt > 0 && C > 0, "bad argument");
    GS_REQ(tex_B == 1 || tex_B == B, "tex batch must be 1 or B");
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t npix = (size_t)B * H * W;
    if (npix == 0) return 0;
    texture_fwd_kernel<<<DR_GRID(npix), 0, s>>>(tex, tex_B, Ht, Wt, C, (const float2*)uv, B, H, W, boundary, out);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int32_t dr_b200_texture_bwd(const float* tex, int32_t tex_B, int32_t Ht, int32_t Wt, int32_t C, const float* uv, int32_t B,
                            int32_t H, int32_t W, int32_t boundary, const float* g_out, float* d_tex, float* d_uv,
                            void* stream) {
    GS_REQ(tex && uv && g_out && d_tex && d_uv, "NULL pointer");
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t npix = (size_t)B * H * W;
    if (npix == 0) return 0;
    texture_bwd_kernel<<<DR_GRID(npix), 0, s>>>(tex, tex_B, Ht, Wt, C, (const float2*)uv, B, H, W, boundary, g_out, d_tex, (float2*)d_uv);
    gs_count_launches(1);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

size_t dr_b200_topology_scratch_bytes(int32_t F) {
    const size_t n = (size_t)3 * F;
    return ((n * 4 + 255) & ~(size_t)255) * 4 + gs_sort_scratch_bytes((int64_t)n) + 256;
}

int32_t dr_b200_edge_opposites(const int32_t* tri, int32_t F, int32_t V, int32_t* opp, void* scratch, void* stream) {
    GS_REQ(F == 0 || (tri && opp && scratch), "NULL pointer");
    const cudaStream_t s = (cudaStream_t)stream;
    if (F <= 0) return 0;
    const int n = 3 * F;
    const size_t stride = ((size_t)n * 4 + 255) & ~(size_t)255;
    char* base = (char*)scratch;
    uint32_t* k0 = (uint32_t*)base; uint32_t* k1 = (uint32_t*)(base + stride);
    uint32_t* v0 = (uint32_t*)(base + 2 * stride); uint32_t* v1 = (uint32_t*)(base + 3 * stride);
    void* sort_scratch = base + 4 * stride;
    int bits = 1; while ((1ll << bits) < (long long)V) bits++;
    topo_emit_kernel<<<DR_GRID(n), 0, s>>>(tri, F, k0, v0);
    int alt = 0;
    if (gs_sort_pairs_u32(k0, k1, v0, v1, n, 0, bits, sort_scratch, &alt, s)) return 1;     // secondary key: max vertex
    uint32_t* vs = alt ? v1 : v0; uint32_t* vo = alt ? v0 : v1;
    uint32_t* ks = alt ? k0 : k1;      // reuse the buffer not holding the sorted keys for the primary keys
    uint32_t* ko = alt ? k1 : k0;
    topo_lo_kernel<<<DR_GRID(n), 0, s>>>(tri, F, vs, ks);
    if (gs_sort_pairs_u32(ks, ko, vs, vo, n, 0, bits, sort_scratch, &alt, s)) return 1;      // primary key: min vertex (stable)
    const uint32_t* sorted_idx = alt ? vo : vs;
    topo_pair_kernel<<<DR_GRID(n), 0, s>>>(tri, F, sorted_idx, opp);
    gs_count_launches(3);
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int32_t dr_b200_antialias_fwd(const float* color, const float* rast, const float* pos, const int32_t* tri, const int32_t* opp,
                              int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t C, float* out, void* stream) {
    GS_REQ(color && rast && out && (F == 0 || (pos && tri && opp)), "NULL pointer");
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t npix = (size_t)B * H * W;
    if (npix == 0) return 0;
    GS_CUDA_CHECK(cudaMemcpyAsync(out, color, npix * C * 4, cudaMemcpyDeviceToDevice, s));
    if (F > 0) {
        antialias_fwd_kernel<<<DR_GRID(npix), 0, s>>>(color, (const float4*)rast, (const float4*)pos, tri, opp, B, V, H, W, C, out);
        gs_count_launches(1);
    }
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}
int32_t dr_b200_antialias_bwd(const float* color, const float* rast, const float* pos, const int32_t* tri, const int32_t* opp,
                              int32_t B, int32_t V, int32_t F, int32_t H, int32_t W, int32_t C, const float* g_out,
                              float* d_color, float* d_pos, void* stream) {
    GS_REQ(color && rast && g_out && d_color && (F == 0 || (pos && tri && opp && d_pos)), "NULL pointer");
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t npix = (size_t)B * H * W;
    if (npix == 0) return 0;
    GS_CUDA_CHECK(cudaMemcpyAsync(d_color, g_out, npix * C * 4, cudaMemcpyDeviceToDevice, s));
    if (F > 0) {
        antialias_bwd_kernel<<<DR_GRID(npix), 0, s>>>(color, (const float4*)rast, (const float4*)pos, tri, opp, B, V, H, W, C, g_out, d_color, d_pos);
        gs_count_launches(1);
    }
    GS_CUDA_CHECK(cudaGetLastError());
    return 0;
}

}  // extern "C"
