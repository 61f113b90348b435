// kintinuous_b200 -- SURF keypoints and descriptors on the device (place recognition, kt_place.cu).
//
// Stands in for cv::SURF(400, 4, 2, false) as backend/PlaceRecognition.cpp:51-88 / DBowInterfaceSurf.cpp:72-99 call it on every keyframe.
// OpenCV's SURF lives in its nonfree module, which is neither in the reference checkout nor installed, so the detector and descriptor are
// restated from the paper (Bay, Ess, Tuytelaars, Van Gool, "Speeded-Up Robust Features", CVIU 110(3), 2008) at the reference's
// parameters, and pinned against the test suite's FP64 numpy restatement of the same steps (tests/test_gpu_place.py):
//   grey      cvtColor(RGB2GRAY) fixed point as OpenCV 4 rounds it: (9798 R + 19235 G + 3735 B + 2^14) >> 15
//   integral  int32, (rows + 1) x (cols + 1), exact
//   Hessian   octave o (4), layer l (4 = 2 + 2): filter side s = (9 + 6 l) << o, lobe L = s / 3, sampled every 2^o pixels;
//             Dxx / Dyy: three L-long lobes (+1 -2 +1) of width 2L - 1, Dxy: four L x L boxes (+ - - +) around a 1-pixel cross;
//             each divided by s^2; det = Dxx Dyy - (0.9 Dxy)^2, laplacian sign = sign(Dxx + Dyy)
//   extrema   det > threshold and strictly greater than its 26 neighbours in (x, y, layer), layers 1 .. 2 of each octave
//   refine    quadratic fit in (x, y, s): offset = -H^-1 g (FP64), kept when every |component| <= 1; size = s + offset_s * 6 << o
//   order     strongest response first, ties by (octave, layer, row, column); the first max_features are described
//   orient    sigma = 1.2 size / 9; the 109 samples (i, j) * sigma with i^2 + j^2 < 36, Haar wavelets of side 2 round(2 sigma),
//             Gaussian weight (2.5 sigma); 72 windows of 60 degrees every 5 degrees; the longest window sum gives the angle
//   describe  20 x 20 samples at sigma spacing in the rotated frame, Haar side 2 round(sigma), Gaussian weight (3.3 sigma), responses
//             rotated into the keypoint frame; 4 x 4 cells of (sum dx, sum dy, sum |dx|, sum |dy|), unit length
// Determinism: every sample of layers 1 .. 2 owns one candidate cell (no capacity, no atomic placement); the cells are sorted by a total
// order (response, octave, layer, position) and every sum has a fixed order, so the output is bitwise reproducible.
#include "kt_ops.h"
#include "../../include/kintinuous_b200.h"
#include <cub/device/device_radix_sort.cuh>

namespace kt {

namespace {

enum { SURF_OCT = 4, SURF_LAY = 4, SCAN_T = 256, DESC_T = 128 };

__device__ __forceinline__ int box_sum(const int* __restrict__ I, int W1, int x0, int y0, int x1, int y1)
{
    return I[y1 * W1 + x1] - I[y0 * W1 + x1] - I[y1 * W1 + x0] + I[y0 * W1 + x0];
}

// grey + row prefix sums: one block per image row; integral row y + 1, column x + 1 = sum of grey[y][0..x]
__global__ void __launch_bounds__(SCAN_T) surf_grey_rows_kernel(const uint8_t* __restrict__ rgb, int rows, int cols, int* __restrict__ I)
{
    __shared__ int s_w[SCAN_T / 32];
    __shared__ int s_carry;
    const int y = blockIdx.x, W1 = cols + 1;
    if (threadIdx.x == 0) { s_carry = 0; I[(y + 1) * W1] = 0; if (y == 0) for (int x = 0; x < W1; ++x) I[x] = 0; }
    __syncthreads();
    for (int base = 0; base < cols; base += SCAN_T) {
        const int x = base + threadIdx.x;
        int g = 0;
        if (x < cols) {
            const uint8_t* p = rgb + ((size_t)y * cols + x) * 3;
            g = (int)((9798u * p[0] + 19235u * p[1] + 3735u * p[2] + (1u << 14)) >> 15);
        }
        int inc = g;
        const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) s_w[wid] = inc;
        __syncthreads();
        int off = s_carry;
        for (int w = 0; w < wid; ++w) off += s_w[w];
        if (x < cols) I[(y + 1) * W1 + x + 1] = off + inc;
        __syncthreads();
        if (threadIdx.x == SCAN_T - 1) { int t = s_carry; for (int w = 0; w < SCAN_T / 32; ++w) t += s_w[w]; s_carry = t; }
        __syncthreads();
    }
}

__global__ void surf_cols_kernel(int rows, int cols, int* __restrict__ I)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, W1 = cols + 1;
    if (x > cols) return;
    int acc = 0;
    for (int y = 1; y <= rows; ++y) { acc += I[y * W1 + x]; I[y * W1 + x] = acc; }
}

// off: each response map's first sample; coff: the first candidate cell of layers 1 and 2 of each octave (one cell per sample of those
// layers, in octave, layer, row, column order), ncells of them
struct SurfGeom { int rows, cols; int grid_r[SURF_OCT], grid_c[SURF_OCT]; size_t off[SURF_OCT][SURF_LAY]; unsigned int coff[SURF_OCT][2]; unsigned int ncells; };

__device__ __forceinline__ int surf_size(int o, int l) { return (9 + 6 * l) << o; }
__device__ __forceinline__ bool surf_fits(int s, int cx, int cy, int rows, int cols)
{
    const int h = s / 2;
    return cx >= h && cy >= h && cx + (s - h) <= cols && cy + (s - h) <= rows;
}

// det of the Hessian (and the laplacian sign in the sign bit of lap) at centre (cx, cy), filter side s; 0 where the filter does not fit
__device__ __forceinline__ float surf_det(const int* __restrict__ I, int W1, int s, int cx, int cy, int* lap)
{
    const int L = s / 3, x0 = cx - s / 2, y0 = cy - s / 2;
    // Dxx: columns x0 + [0, s) in three lobes, rows cy - (L - 1) .. cy + L - 1
    const int ya = cy - (L - 1), yb = cy + L;
    const int xx = box_sum(I, W1, x0, ya, x0 + s, yb) - 3 * box_sum(I, W1, x0 + L, ya, x0 + 2 * L, yb);
    const int xa = cx - (L - 1), xb = cx + L;
    const int yy = box_sum(I, W1, xa, y0, xb, y0 + s) - 3 * box_sum(I, W1, xa, y0 + L, xb, y0 + 2 * L);
    const int xy = box_sum(I, W1, cx - L, cy - L, cx, cy) - box_sum(I, W1, cx + 1, cy - L, cx + 1 + L, cy)
                 - box_sum(I, W1, cx - L, cy + 1, cx, cy + 1 + L) + box_sum(I, W1, cx + 1, cy + 1, cx + 1 + L, cy + 1 + L);
    const float inv = __fdiv_rn(1.0f, (float)(s * s));          // IEEE: the build's --prec-div=false would approximate it
    const float dxx = (float)xx * inv, dyy = (float)yy * inv, dxy = (float)xy * inv;
    *lap = (xx + yy) >= 0 ? 1 : -1;
    return __fsub_rn(__fmul_rn(dxx, dyy), __fmul_rn(0.81f, __fmul_rn(dxy, dxy)));
}

// every octave / layer response map in one launch: blockIdx.y = o * 4 + l
__global__ void surf_hessian_kernel(const int* __restrict__ I, const SurfGeom g, float* __restrict__ resp)
{
    const int o = blockIdx.y / SURF_LAY, l = blockIdx.y % SURF_LAY;
    const int gc = g.grid_c[o], gr = g.grid_r[o];
    const int n = gr * gc, s = surf_size(o, l), W1 = g.cols + 1;
    float* out = resp + g.off[o][l];
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const int i = k / gc, j = k - i * gc, cx = j << o, cy = i << o;
        int lap;
        out[k] = surf_fits(s, cx, cy, g.rows, g.cols) ? surf_det(I, W1, s, cx, cy, &lap) : 0.f;
    }
}

struct SurfCand { unsigned long long key; float x, y, size, response; int lap; int pad; };

__device__ __forceinline__ unsigned int ord_desc(float f)     // larger float -> smaller key
{
    const unsigned int u = __float_as_uint(f);
    const unsigned int o = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ~o;
}

// 3 x 3 x 3 maxima of layers 1 .. 2 above the threshold, refined by the quadratic fit; blockIdx.y = o * 2 + (l - 1).  Every sample owns
// one candidate cell (so there is no capacity to overflow and no atomic decides where a candidate lands): its sort key is (response
// descending, cell index) for an extremum and ~0 otherwise; the atomic counter only counts the extrema.
__global__ void surf_extrema_kernel(const int* __restrict__ I, const SurfGeom g, const float* __restrict__ resp, float threshold,
                                    SurfCand* __restrict__ cand, unsigned long long* __restrict__ keys, unsigned int* __restrict__ idx,
                                    unsigned int* __restrict__ n_cand)
{
    const int o = blockIdx.y / 2, l = 1 + blockIdx.y % 2;
    const int gc = g.grid_c[o], gr = g.grid_r[o], n = gr * gc;
    const float* R0 = resp + g.off[o][l - 1]; const float* R1 = resp + g.off[o][l]; const float* R2 = resp + g.off[o][l + 1];
    const int s_hi = surf_size(o, l + 1);
    const unsigned int cb = g.coff[o][l - 1];
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        keys[cb + k] = ~0ull; idx[cb + k] = cb + k;
        const int i = k / gc, j = k - i * gc;
        if (i < 1 || j < 1 || i >= gr - 1 || j >= gc - 1) continue;
        const float v = R1[k];
        if (!(v > threshold)) continue;
        // every neighbour must be a real response: the largest filter fits at the four corner neighbours
        if (!surf_fits(s_hi, (j - 1) << o, (i - 1) << o, g.rows, g.cols) || !surf_fits(s_hi, (j + 1) << o, (i + 1) << o, g.rows, g.cols)) continue;
        bool mx = true;
        for (int dy = -1; dy <= 1 && mx; ++dy)
            for (int dx = -1; dx <= 1; ++dx) {
                const int q = k + dy * gc + dx;
                if (R0[q] >= v || R2[q] >= v || ((dx || dy) && R1[q] >= v)) { mx = false; break; }
            }
        if (!mx) continue;
        // quadratic fit: gradient and Hessian by central differences over (x, y, layer), FP64
        const double dx = 0.5 * ((double)R1[k + 1] - R1[k - 1]), dy = 0.5 * ((double)R1[k + gc] - R1[k - gc]), ds = 0.5 * ((double)R2[k] - R0[k]);
        const double c2 = 2.0 * v;
        const double hxx = (double)R1[k + 1] + R1[k - 1] - c2, hyy = (double)R1[k + gc] + R1[k - gc] - c2, hss = (double)R2[k] + R0[k] - c2;
        const double hxy = 0.25 * ((double)R1[k + gc + 1] - R1[k + gc - 1] - R1[k - gc + 1] + R1[k - gc - 1]);
        const double hxs = 0.25 * ((double)R2[k + 1] - R2[k - 1] - R0[k + 1] + R0[k - 1]);
        const double hys = 0.25 * ((double)R2[k + gc] - R2[k - gc] - R0[k + gc] + R0[k - gc]);
        const double det = hxx * (hyy * hss - hys * hys) - hxy * (hxy * hss - hys * hxs) + hxs * (hxy * hys - hyy * hxs);
        if (det == 0.0) continue;
        // offset = -H^-1 g (Cramer)
        const double ox = -(dx * (hyy * hss - hys * hys) - hxy * (dy * hss - hys * ds) + hxs * (dy * hys - hyy * ds)) / det;
        const double oy = -(hxx * (dy * hss - ds * hys) - dx * (hxy * hss - hys * hxs) + hxs * (hxy * ds - dy * hxs)) / det;
        const double os = -(hxx * (hyy * ds - hys * dy) - hxy * (hxy * ds - hxs * dy) + dx * (hxy * hys - hyy * hxs)) / det;
        if (fabs(ox) > 1.0 || fabs(oy) > 1.0 || fabs(os) > 1.0) continue;
        int lap;
        surf_det(I, g.cols + 1, surf_size(o, l), j << o, i << o, &lap);
        atomicAdd(n_cand, 1u);
        SurfCand c;
        c.key = ((unsigned long long)ord_desc(v) << 32) | (unsigned long long)(cb + k);
        c.x = (float)(((double)j + ox) * (double)(1 << o)); c.y = (float)(((double)i + oy) * (double)(1 << o));
        c.size = (float)((double)surf_size(o, l) + os * (double)(6 << o));
        c.response = v; c.lap = lap; c.pad = 0;
        cand[cb + k] = c; keys[cb + k] = c.key;
    }
}

// Haar wavelet responses of side hs (even) centred on pixel (px, py): dx = right - left, dy = bottom - top; false outside the image
__device__ __forceinline__ bool haar(const int* __restrict__ I, int W1, int rows, int cols, int px, int py, int hs, float* dx, float* dy)
{
    const int h = hs / 2, x0 = px - h, y0 = py - h;
    if (x0 < 0 || y0 < 0 || x0 + hs > cols || y0 + hs > rows) return false;
    *dx = (float)(box_sum(I, W1, px, y0, x0 + hs, y0 + hs) - box_sum(I, W1, x0, y0, px, y0 + hs));
    *dy = (float)(box_sum(I, W1, x0, py, x0 + hs, y0 + hs) - box_sum(I, W1, x0, y0, x0 + hs, py));
    return true;
}

// one block per kept keypoint: orientation, then the 64-d descriptor; kp: x, y, size, angle (radians), response, laplacian
__global__ void __launch_bounds__(DESC_T) surf_describe_kernel(const int* __restrict__ I, int rows, int cols, const SurfCand* __restrict__ cand,
                                                               const unsigned int* __restrict__ order, const unsigned int* __restrict__ n_cand,
                                                               int max_features, float* __restrict__ kp, float* __restrict__ desc,
                                                               int* __restrict__ n_out)
{
    __shared__ float s_dx[400], s_dy[400], s_ang[112];
    __shared__ float s_win[72];
    __shared__ float s_cell[64];
    __shared__ float s_theta;
    const int n = (int)min(*n_cand, (unsigned int)max_features);
    if (blockIdx.x == 0 && threadIdx.x == 0) *n_out = n;
    if ((int)blockIdx.x >= n) return;
    const SurfCand c = cand[order[blockIdx.x]];
    const int W1 = cols + 1;
    const float sigma = __fdiv_rn(__fmul_rn(1.2f, c.size), 9.0f);
    // orientation samples
    const int hs_o = 2 * max(1, __float2int_rn(2.0f * sigma));
    for (int t = threadIdx.x; t < 169; t += DESC_T) {
        const int i = t % 13 - 6, j = t / 13 - 6;
        // compact index of (i, j) among the 109 disc samples in row-major (j, i) order
        if (i * i + j * j >= 36) continue;
        int slot = 0;
        for (int jj = -6; jj < j; ++jj) for (int ii = -6; ii <= 6; ++ii) slot += (ii * ii + jj * jj < 36) ? 1 : 0;
        for (int ii = -6; ii < i; ++ii) slot += (ii * ii + j * j < 36) ? 1 : 0;
        float dx = 0.f, dy = 0.f;
        const int px = __float2int_rn(c.x + (float)i * sigma), py = __float2int_rn(c.y + (float)j * sigma);
        if (haar(I, W1, rows, cols, px, py, hs_o, &dx, &dy)) {
            const float w = expf(-(float)(i * i + j * j) / (2.0f * 2.5f * 2.5f));
            dx *= w; dy *= w;
        } else { dx = 0.f; dy = 0.f; }
        s_dx[slot] = dx; s_dy[slot] = dy;
        float a = atan2f(dy, dx) * 57.29577951308232f;
        if (a < 0.f) a += 360.f;
        s_ang[slot] = (dx == 0.f && dy == 0.f) ? -1000.f : a;
    }
    __syncthreads();
    if (threadIdx.x < 72) {
        const float ori = 5.0f * (float)threadIdx.x;
        float sx = 0.f, sy = 0.f;
        for (int k = 0; k < 109; ++k) {
            if (s_ang[k] < -999.f) continue;
            const float d = fabsf(s_ang[k] - ori);
            if (d < 30.f || d > 330.f) { sx += s_dx[k]; sy += s_dy[k]; }
        }
        s_win[threadIdx.x] = sx * sx + sy * sy;
        s_dx[200 + threadIdx.x] = sx; s_dy[200 + threadIdx.x] = sy;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int b = 0;
        for (int k = 1; k < 72; ++k) if (s_win[k] > s_win[b]) b = k;
        s_theta = atan2f(s_dy[200 + b], s_dx[200 + b]);
    }
    __syncthreads();
    const float th = s_theta, co = cosf(th), si = sinf(th);
    const int hs_d = 2 * max(1, __float2int_rn(sigma));
    const float inv2s = 1.0f / (2.0f * 3.3f * 3.3f * sigma * sigma);
    for (int t = threadIdx.x; t < 400; t += DESC_T) {
        const int u = t % 20, v = t / 20;
        const float ox = ((float)u - 9.5f) * sigma, oy = ((float)v - 9.5f) * sigma;
        const int px = __float2int_rn(c.x + co * ox - si * oy), py = __float2int_rn(c.y + si * ox + co * oy);
        float dx = 0.f, dy = 0.f;
        if (haar(I, W1, rows, cols, px, py, hs_d, &dx, &dy)) {
            const float w = expf(-(ox * ox + oy * oy) * inv2s);
            const float rx = (dx * co + dy * si) * w, ry = (-dx * si + dy * co) * w;
            dx = rx; dy = ry;
        }
        s_dx[t] = dx; s_dy[t] = dy;
    }
    __syncthreads();
    if (threadIdx.x < 64) {
        const int cell = threadIdx.x >> 2, comp = threadIdx.x & 3, cu = cell & 3, cv = cell >> 2;
        float acc = 0.f;
        for (int v = 0; v < 5; ++v)
            for (int u = 0; u < 5; ++u) {
                const int t = (cv * 5 + v) * 20 + cu * 5 + u;
                const float a = (comp & 1) ? s_dy[t] : s_dx[t];
                acc += comp >= 2 ? fabsf(a) : a;
            }
        s_cell[threadIdx.x] = acc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float ss = 0.f;
        for (int k = 0; k < 64; ++k) ss += s_cell[k] * s_cell[k];
        s_win[0] = ss > 0.f ? 1.0f / sqrtf(ss) : 0.f;
        float* o = kp + (size_t)blockIdx.x * 6;
        o[0] = c.x; o[1] = c.y; o[2] = c.size; o[3] = th; o[4] = c.response; o[5] = (float)c.lap;
    }
    __syncthreads();
    if (threadIdx.x < 64) desc[(size_t)blockIdx.x * 64 + threadIdx.x] = s_cell[threadIdx.x] * s_win[0];
}

} // namespace

static SurfGeom surf_geom(int rows, int cols)
{
    SurfGeom g; g.rows = rows; g.cols = cols;
    size_t off = 0;
    for (int o = 0; o < SURF_OCT; ++o) {
        const int step = 1 << o;
        g.grid_r[o] = (rows + step - 1) / step; g.grid_c[o] = (cols + step - 1) / step;
        for (int l = 0; l < SURF_LAY; ++l) { g.off[o][l] = off; off += (size_t)g.grid_r[o] * g.grid_c[o]; }
    }
    size_t c = 0;
    for (int o = 0; o < SURF_OCT; ++o) for (int l = 0; l < 2; ++l) { g.coff[o][l] = (unsigned int)c; c += (size_t)g.grid_r[o] * g.grid_c[o]; }
    g.ncells = (unsigned int)c;
    return g;
}

int surf_ws_reserve(SurfWorkspace* ws, int rows, int cols)
{
    if (ws->rows == rows && ws->cols == cols) return 0;
    *ws = SurfWorkspace();
    const SurfGeom g = surf_geom(rows, cols);
    size_t nresp = 0;
    for (int o = 0; o < SURF_OCT; ++o) nresp += (size_t)SURF_LAY * g.grid_r[o] * g.grid_c[o];
    const size_t nc = g.ncells;
    size_t tmp = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp, (unsigned long long*)0, (unsigned long long*)0, (unsigned int*)0, (unsigned int*)0, (int)nc);
    SurfCand* cand = 0;
    int r;
    if ((r = ws->mem.device(&ws->integral, (size_t)(rows + 1) * (cols + 1), "surf integral image")) ||
        (r = ws->mem.device(&ws->resp, nresp, "surf responses")) || (r = ws->mem.device(&cand, nc, "surf candidates")) ||
        (r = ws->mem.device(&ws->keys, nc * 2, "surf sort keys")) || (r = ws->mem.device(&ws->idx, nc * 2, "surf sort indices")) ||
        (r = ws->mem.device(&ws->n_cand, 1, "surf candidate count")) || (r = ws->mem.device(&ws->tmp, tmp, "surf sort storage"))) return r;
    ws->cand = cand; ws->tmp_bytes = tmp; ws->rows = rows; ws->cols = cols;
    return 0;
}

int surf(const uint8_t* rgb, int rows, int cols, float threshold, int max_features, float* kp, float* desc, int* n_out, SurfWorkspace* ws, cudaStream_t s)
{
    if (rows < 32 || cols < 32 || max_features < 1) { set_error("surf: the image must be at least 32 x 32 and max_features >= 1"); return KT_ERR_INVALID; }
    int r = surf_ws_reserve(ws, rows, cols); if (r) return r;
    const SurfGeom g = surf_geom(rows, cols);
    surf_grey_rows_kernel<<<rows, SCAN_T, 0, s>>>(rgb, rows, cols, ws->integral);
    KT_LAUNCH_CHECK();
    surf_cols_kernel<<<div_up(cols + 1, 128), 128, 0, s>>>(rows, cols, ws->integral);
    KT_LAUNCH_CHECK();
    const int sms = device_info().sm_count;
    surf_hessian_kernel<<<dim3(sms * 2, SURF_OCT * SURF_LAY), 256, 0, s>>>(ws->integral, g, ws->resp);
    KT_LAUNCH_CHECK();
    KT_CUDA(cudaMemsetAsync(ws->n_cand, 0, sizeof(unsigned int), s));
    const size_t nc = g.ncells;
    unsigned long long* keys_in = ws->keys; unsigned long long* keys_out = ws->keys + nc;
    unsigned int* idx_in = ws->idx; unsigned int* idx_out = ws->idx + nc;
    surf_extrema_kernel<<<dim3(sms, SURF_OCT * 2), 256, 0, s>>>(ws->integral, g, ws->resp, threshold, (SurfCand*)ws->cand, keys_in, idx_in, ws->n_cand);
    KT_LAUNCH_CHECK();
    size_t tmp = ws->tmp_bytes;
    KT_CUDA(cub::DeviceRadixSort::SortPairs(ws->tmp, tmp, keys_in, keys_out, idx_in, idx_out, (int)nc, 0, 64, s));
    ++g_launches;
    surf_describe_kernel<<<max_features, DESC_T, 0, s>>>(ws->integral, rows, cols, (const SurfCand*)ws->cand, idx_out, ws->n_cand,
                                                         max_features, kp, desc, n_out);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
