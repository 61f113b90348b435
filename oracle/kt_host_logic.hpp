// TEST INFRASTRUCTURE ONLY (oracle/): never linked into, imported by or executed from the
// product path (kintinuous_b200/).
//
// Restatement of the reference's HOST control flow for the per-frame tracking-and-fusion path,
// templated on a Backend that supplies the operators of src/frontend/cuda/internal.h:299-536.
// Two backends instantiate it:
//   * oracle/kt_oracle_cpu.cpp  -- CPU restatement of every kernel ("port" oracle)
//   * oracle/ref_harness.cu     -- the reference's own, unmodified CUDA operators compiled from
//                                  the reference checkout (oracle/_ref/libkt_ref_<VOL>.so, "reference" oracle)
// so both run the *same* host logic; the reference host classes themselves cannot be compiled
// here (they need Eigen/OpenCV/PCL/Boost, none installed -- SURVEY.md D6).
//
// Follows, line by line where it matters:
//   KintinuousTracker::KintinuousTracker   KintinuousTracker.cpp:71-182   (volumeBasis, trunc dist)
//   KintinuousTracker::reset               KintinuousTracker.cpp:262-354
//   KintinuousTracker::processFrame        KintinuousTracker.cpp:444-915
//   KintinuousTracker::vWrapCopyUpdate     KintinuousTracker.cpp:1075-1085
//   KintinuousTracker::mutexOutCloudBuffer KintinuousTracker.cpp:1156-1208
//   KintinuousTracker::finalise            KintinuousTracker.cpp:1003-1048
//   TsdfVolume::setTsdfTruncDist           TSDFVolume.cpp:89-97
//   ICPOdometry::getIncrementalTransformation   ICPOdometry.cpp:68-186
//   RGBDOdometry::getIncrementalTransformation  RGBDOdometry.cpp:165-393 (+ populateRGBDData :140-163)
// Out of scope (SURVEY.md §2): place recognition, dynamicCube, ground-truth odometry, GUI taps,
// .poses file I/O (Q14).
#pragma once
#include <vector>
#include <cstdint>
#include <cstdio>
#include <cmath>
#include <climits>
#include <algorithm>
#include "kt_hostmath.hpp"

namespace kto {

struct IntrF { float fx, fy, cx, cy;
    IntrF level(int l) const { int d = 1 << l; IntrF r = {fx / d, fy / d, cx / d, cy / d}; return r; } };  // internal.h:255-259
struct IntrD { double fx, fy, cx, cy;
    IntrD level(int l) const { int d = 1 << l; IntrD r = {fx / d, fy / d, cx / d, cy / d}; return r; } };  // internal.h:268-272

struct PointXYZRGB32 { float x, y, z, pad; unsigned char b, g, r, a; unsigned char pad2[12]; };  // internal.h:156-184 (32 B)
static_assert(sizeof(PointXYZRGB32) == 32, "PointXYZRGB must be 32 bytes");

enum SliceDim { XPlus = 0, XMinus, YPlus, YMinus, ZPlus, ZMinus, FIRST, FINAL_, TSDF_ };  // CloudSlice.h:33-44 order

struct Slice {
    int dimension;
    std::vector<PointXYZRGB32> points;
    float camera_t[3];     // currentGlobalCamera at hand-off
    float camera_R[9];
    uint64_t utime;
};

struct TrackerConfig {
    int rows, cols;
    float fx, fy, cx, cy;
    int vol;                 // voxels per side (must equal the backend's compile-time VOL for the CUDA reference)
    float volume_size;       // metres (ConfigArgs -s, default 6)
    int odometry;            // 0 = ICP (default), 1 = RGB-D only (-r), 2 = ICP+RGB-D (-ri)
    int fast_odometry;       // -fod
    int voxel_shift;         // -t, default 14
    int overlap;             // TrackerInterface.h:58 default 2
    int angle_color;         // !disableColorAngleWeight (-dc), default 1
    int parked;              // staticMode-like: never shift
    int cloud_capacity;      // points; reference: 3*rows*cols (KintinuousTracker.cpp:77)
};

template <class B>
class RefTracker {
public:
    static const int LEVELS = 4;      // ICPOdometry.h:52, RGBDOdometry.h:96

    RefTracker(B& backend, const TrackerConfig& c) : be(backend), cfg(c)
    {
        intr.fx = c.fx; intr.fy = c.fy; intr.cx = c.cx; intr.cy = c.cy;
        intrD.fx = intr.fx; intrD.fy = intr.fy; intrD.cx = intr.cx; intrD.cy = intr.cy;   // RGBDOdometry.cpp:70-73 (from float Intr)
        size = c.volume_size;
        voxel = size / (float)c.vol;                       // Volume.h:46-48, TSDFVolume.cpp:119-123
        // KintinuousTracker.cpp:112-113 + TSDFVolume.cpp:89-97
        float def = std::max(0.01f, size / 100.0f);
        trunc = std::max(def, 2.1f * voxel);
        volumeBasis[0] = volumeBasis[1] = volumeBasis[2] = size * 0.5f;                    // :109 (non-static mode)
        size_t P = (size_t)c.rows * c.cols;
        size_t V = (size_t)c.vol * c.vol * c.vol;
        tsdf = (short*)be.alloc(V * sizeof(short));
        color = (unsigned char*)be.alloc(V * 4);
        for (int l = 0; l < LEVELS; ++l) {
            size_t Pl = P >> (2 * l);
            depths_curr[l] = (uint16_t*)be.alloc(Pl * 2);
            vmaps_g_prev[l] = (float*)be.alloc(Pl * 12);  nmaps_g_prev[l] = (float*)be.alloc(Pl * 12);
            vmaps_curr[l] = (float*)be.alloc(Pl * 12);    nmaps_curr[l] = (float*)be.alloc(Pl * 12);
            // Q7: invalid pixels leave stale y/z planes; make the stale content deterministic (zeros).
            be.zero(vmaps_g_prev[l], Pl * 12); be.zero(nmaps_g_prev[l], Pl * 12);
            be.zero(vmaps_curr[l], Pl * 12);   be.zero(nmaps_curr[l], Pl * 12);
        }
        vmap_curr_color = (unsigned char*)be.alloc(P * 4); be.zero(vmap_curr_color, P * 4);
        depthRawScaled = (float*)be.alloc(P * 4);
        depth_raw = (uint16_t*)be.alloc(P * 2);
        rgb = (unsigned char*)be.alloc(P * 3);
        cloud_device = (PointXYZRGB32*)be.alloc((size_t)c.cloud_capacity * sizeof(PointXYZRGB32));
        if (c.odometry != 0) {
            for (int l = 0; l < LEVELS; ++l) {
                size_t Pl = P >> (2 * l);
                lastDepth[l] = (float*)be.alloc(Pl * 4); nextDepth[l] = (float*)be.alloc(Pl * 4);
                lastImage[l] = (unsigned char*)be.alloc(Pl); nextImage[l] = (unsigned char*)be.alloc(Pl);
                nextdIdx[l] = (short*)be.alloc(Pl * 2); nextdIdy[l] = (short*)be.alloc(Pl * 2);
                pointClouds[l] = (float*)be.alloc(Pl * 12);
                corresImg[l] = be.alloc(Pl * 16);
            }
        }
        // ICPOdometry.cpp:42-55 / RGBDOdometry.cpp:76-107
        if (c.odometry == 1) { int it[4] = {10, 7, 7, 7}; int itf[4] = {0, 10, 7, 0}; for (int i = 0; i < 4; ++i) iterations[i] = c.fast_odometry ? itf[i] : it[i]; }
        else if (c.odometry == 2) { int it[4] = {10, 5, 4, 0}; int itf[4] = {0, 10, 7, 0}; for (int i = 0; i < 4; ++i) iterations[i] = c.fast_odometry ? itf[i] : it[i]; }
        else { int it[4] = {10, 5, 4, 0}; int itf[4] = {0, 10, 5, 0}; for (int i = 0; i < 4; ++i) iterations[i] = c.fast_odometry ? itf[i] : it[i]; }
        reset();
    }

    ~RefTracker()
    {
        be.free(tsdf); be.free(color);
        for (int l = 0; l < LEVELS; ++l) {
            be.free(depths_curr[l]); be.free(vmaps_g_prev[l]); be.free(nmaps_g_prev[l]); be.free(vmaps_curr[l]); be.free(nmaps_curr[l]);
            if (cfg.odometry != 0) {
                be.free(lastDepth[l]); be.free(nextDepth[l]); be.free(lastImage[l]); be.free(nextImage[l]);
                be.free(nextdIdx[l]); be.free(nextdIdy[l]); be.free(pointClouds[l]); be.free(corresImg[l]);
            }
        }
        be.free(vmap_curr_color); be.free(depthRawScaled); be.free(depth_raw); be.free(rgb); be.free(cloud_device);
    }

    void reset()                                           // KintinuousTracker.cpp:262-354
    {
        global_time = 0;
        rmats.clear(); tvecs.clear();
        rmats.push_back(mat3_identity());
        Vec3f tb = {{volumeBasis[0], volumeBasis[1], volumeBasis[2]}};
        tvecs.push_back(tb);
        voxelWrap[0] = voxelWrap[1] = voxelWrap[2] = 0;
        for (int i = 0; i < 3; ++i) currentGlobalCamera[i] = volumeBasis[i] - size * 0.5f;
        slices.clear();
        be.init_volume(tsdf, color, cfg.vol);
        icp_iters_done = 0;
    }

    // One frame. depth_host: rows*cols u16 (mm); rgb_host: rows*cols*3 u8 (PixelRGB r,g,b).
    // The upload is what TrackerInterface.cpp:90-91 does before calling processFrame.
    void processFrame(const uint16_t* depth_host, const unsigned char* rgb_host, uint64_t timestamp)
    {
        const int rows = cfg.rows, cols = cfg.cols;
        const size_t P = (size_t)rows * cols;
        be.upload(depth_raw, depth_host, P * 2);
        be.upload(rgb, rgb_host, P * 3);

        const bool use_icp_maps = (cfg.odometry == 0) || (cfg.odometry == 2) || cfg.angle_color;     // :465 (Q10)
        if (use_icp_maps) {
            be.bilateral(depth_raw, depths_curr[0], rows, cols);                                      // :467
            for (int i = 1; i < LEVELS; ++i) be.pyrdown(depths_curr[i-1], depths_curr[i], rows >> (i-1), cols >> (i-1));
            for (int i = 0; i < LEVELS; ++i) {
                be.vmap(depths_curr[i], vmaps_curr[i], rows >> i, cols >> i, intr.level(i));
                be.nmap(vmaps_curr[i], nmaps_curr[i], rows >> i, cols >> i);
            }
        }

        float vol_size3[3] = {size, size, size};

        if (global_time == 0) {                                                                      // :481-557
            Mat3f Rcam = rmats.back(); Vec3f tcam = tvecs.back();
            Mat3f Rcam_inv = mat3_inverse_eigen(Rcam);
            int emptyVoxel[3] = {0, 0, 0};
            if (cfg.odometry != 0) populateRGBDData(depth_raw, rgb, lastDepth, lastImage);           // rgbd->firstRun :499-502
            be.integrate(depth_raw, rows, cols, intr, vol_size3, Rcam_inv.m, tcam.v, trunc, tsdf, color, cfg.vol,
                         emptyVoxel, rgb, nmaps_curr[0], cfg.angle_color, depthRawScaled);
            for (int i = 0; i < LEVELS; ++i)
                be.transform_maps(vmaps_curr[i], nmaps_curr[i], Rcam.m, tcam.v, vmaps_g_prev[i], nmaps_g_prev[i], rows >> i, cols >> i);
            ++global_time;
            current_utime = timestamp;
            return;
        }

        Mat3f Rprev = rmats.back(); Vec3f tprev = tvecs.back();
        Mat3f Rcurr = Rprev; Vec3f tcurr = tprev;

        if (cfg.odometry == 0) icpOdometry(Rprev, tprev, &Rcurr, &tcurr);
        else rgbdOdometry(Rprev, tprev, &Rcurr, &tcurr);

        current_utime = timestamp;
        rmats.push_back(Rcurr); tvecs.push_back(tcurr);                                              // :578-579

        // :581-596 currentGlobalCamera
        for (int i = 0; i < 3; ++i) {
            float initialTrans = volumeBasis[i] - size * 0.5f;
            float g = initialTrans;
            g += voxelWrap[i] * voxel;
            g += tcurr.v[i] - volumeBasis[i];
            currentGlobalCamera[i] = g;
        }

        Mat3f Rcurr_inv = mat3_inverse_eigen(Rcurr);                                                 // :627
        float currentTranslation[3];
        for (int i = 0; i < 3; ++i) currentTranslation[i] = tvecs.back().v[i] - volumeBasis[i];      // :632
        const int thresh = cfg.parked ? INT_MAX : cfg.voxel_shift;                                  // :636
        int trans[3];
        for (int i = 0; i < 3; ++i) {                                                                // :642-667
            int f = (int)std::floor(currentTranslation[i] / voxel);
            trans[i] = (f < 0) ? std::max(-thresh, f) : std::min(thresh, f);
        }
        const int V = cfg.vol;
        int vWrapCopy[3];
        for (int axis = 0; axis < 3; ++axis) {                                                       // x :675-723, y :729-777, z :783-831
            vWrapCopyUpdate(vWrapCopy);
            bool cycled = false;
            int lo[3] = {0, 0, 0}, hi[3] = {V, V, V};
            const int n = trans[axis];
            if (n >= thresh) {
                lo[axis] = 0; hi[axis] = n + 1 + cfg.overlap;
                fetchCloud(vWrapCopy, lo, hi);
                be.clear(axis, 0, tsdf, color, V, voxelWrap[axis], voxelWrap[axis] + n);
                cycled = true;
            } else if (n <= -thresh) {
                if (axis < 2) { lo[axis] = V + (n - cfg.overlap); hi[axis] = V; }
                else          { lo[axis] = V + (n - cfg.overlap) - 1; hi[axis] = V - 1; }            // :805 (Q12)
                fetchCloud(vWrapCopy, lo, hi);
                be.clear(axis, 1, tsdf, color, V, voxelWrap[axis], voxelWrap[axis] + n);
                cycled = true;
            }
            if (cycled) {
                int vt[3] = {0, 0, 0}; vt[axis] = n;
                mutexOutCloudBuffer(&tcurr, vt);
            }
        }
        vWrapCopyUpdate(vWrapCopy);

        be.integrate(depth_raw, rows, cols, intr, vol_size3, Rcurr_inv.m, tcurr.v, trunc, tsdf, color, cfg.vol,
                     vWrapCopy, rgb, nmaps_curr[0], cfg.angle_color, depthRawScaled);                // :864-876
        vWrapCopyUpdate(vWrapCopy);
        be.raycast(intr, Rcurr.m, tcurr.v, trunc, vol_size3, tsdf, cfg.vol, vmaps_g_prev[0], nmaps_g_prev[0], rows, cols,
                   vWrapCopy, vmap_curr_color, color);                                               // :880-890
        if (cfg.odometry == 0 || cfg.odometry == 2) {                                                // :892-899
            for (int i = 1; i < LEVELS; ++i) {
                be.resize_vmap(vmaps_g_prev[i-1], vmaps_g_prev[i], rows >> (i-1), cols >> (i-1));
                be.resize_nmap(nmaps_g_prev[i-1], nmaps_g_prev[i], rows >> (i-1), cols >> (i-1));
            }
        }
        ++global_time;
    }

    void finalise()                                                                                  // :1003-1048
    {
        int vWrapCopy[3]; vWrapCopyUpdate(vWrapCopy);
        const int V = cfg.vol;
        int lo[3] = {0, 0, 0}, hi[3] = {V, V, V};
        fetchCloud(vWrapCopy, lo, hi);
        Slice s; s.dimension = FINAL_;
        s.points.resize(cloud_count);
        if (cloud_count) be.download(s.points.data(), cloud_device, cloud_count * sizeof(PointXYZRGB32));
        for (int i = 0; i < 3; ++i) s.camera_t[i] = currentGlobalCamera[i];
        for (int i = 0; i < 9; ++i) s.camera_R[i] = rmats.back().m[i];
        s.utime = current_utime;
        slices.push_back(std::move(s));
    }

    // ---- state exposed to the C wrappers ----
    B& be; TrackerConfig cfg;
    IntrF intr; IntrD intrD;
    float size, voxel, trunc;
    float volumeBasis[3];
    float currentGlobalCamera[3];
    int voxelWrap[3];
    int global_time; uint64_t current_utime = 0;
    std::vector<Mat3f> rmats; std::vector<Vec3f> tvecs;
    std::vector<Slice> slices;
    short* tsdf; unsigned char* color;
    uint16_t* depths_curr[LEVELS]; float* vmaps_g_prev[LEVELS]; float* nmaps_g_prev[LEVELS]; float* vmaps_curr[LEVELS]; float* nmaps_curr[LEVELS];
    unsigned char* vmap_curr_color; float* depthRawScaled; uint16_t* depth_raw; unsigned char* rgb;
    PointXYZRGB32* cloud_device; size_t cloud_count = 0;
    float* lastDepth[LEVELS]; float* nextDepth[LEVELS]; unsigned char* lastImage[LEVELS]; unsigned char* nextImage[LEVELS];
    short* nextdIdx[LEVELS]; short* nextdIdy[LEVELS]; float* pointClouds[LEVELS]; void* corresImg[LEVELS];
    int iterations[LEVELS];
    // per-iteration trace of the last frame (for golden vectors): A(36) b(6) residual(2) per iteration
    std::vector<float> trace;
    int icp_iters_done;

    void vWrapCopyUpdate(int* w) const                                                               // :1075-1085
    {
        const int V = cfg.vol;
        for (int i = 0; i < 3; ++i) { w[i] = voxelWrap[i]; if (w[i] < 0) w[i] = V - ((-w[i]) % V); }
    }

private:
    void fetchCloud(const int* vWrapCopy, const int* lo, const int* hi)                              // TSDFVolume.cpp:131-172
    {
        float vol_size3[3] = {size, size, size};
        cloud_count = be.extract(tsdf, vol_size3, cfg.vol, cloud_device, (size_t)cfg.cloud_capacity, vWrapCopy, color,
                                 lo[0], hi[0], lo[1], hi[1], lo[2], hi[2], 1, voxelWrap);
    }

    void mutexOutCloudBuffer(Vec3f* device_tcurr, const int* vt)                                     // :1156-1208
    {
        Slice s;
        s.points.resize(cloud_count);
        if (cloud_count) be.download(s.points.data(), cloud_device, cloud_count * sizeof(PointXYZRGB32));
        float voxelTransSize[3];
        for (int i = 0; i < 3; ++i) voxelTransSize[i] = voxel * vt[i];
        for (int i = 0; i < 3; ++i) tvecs.back().v[i] -= voxelTransSize[i];
        s.dimension = vt[0] > 0 ? XPlus : vt[0] < 0 ? XMinus : vt[1] > 0 ? YPlus : vt[1] < 0 ? YMinus : vt[2] > 0 ? ZPlus : ZMinus;
        for (int i = 0; i < 3; ++i) s.camera_t[i] = currentGlobalCamera[i];
        for (int i = 0; i < 9; ++i) s.camera_R[i] = rmats.back().m[i];
        s.utime = current_utime;
        slices.push_back(std::move(s));
        for (int i = 0; i < 3; ++i) voxelWrap[i] += vt[i];
        for (int i = 0; i < 3; ++i) device_tcurr->v[i] -= voxelTransSize[i];
    }

    void solveAndUpdate(const double* dA, const double* db, double* resultRt, const Mat3f& Rprev, const Vec3f& tprev,
                        Mat3f* Rcurr, Vec3f* tcurr)
    {
        double result[6];
        ldlt6_solve(dA, db, result);                                       // ICPOdometry.cpp:131
        double currRt[16], tmp[16];
        projective_matrix(result, currRt);                                 // :142
        mat4d_mul(currRt, resultRt, tmp);                                  // :144
        for (int k = 0; k < 16; ++k) resultRt[k] = tmp[k];
        compose_prev_with_inverse(Rprev, tprev, resultRt, Rcurr, tcurr);   // :146-178
    }

    void icpOdometry(const Mat3f& Rprev, const Vec3f& tprev, Mat3f* Rcurr, Vec3f* tcurr)             // ICPOdometry.cpp:68-186
    {
        Mat3f Rprev_inv = mat3_inverse_eigen(Rprev);
        double resultRt[16]; for (int k = 0; k < 16; ++k) resultRt[k] = (k % 5 == 0) ? 1.0 : 0.0;
        trace.clear(); icp_iters_done = 0;
        const float distThres = 0.10f, angleThres = sinf(20.f * 3.14159254f / 180.f);               // ICPOdometry.h:35-36
        for (int level = LEVELS - 1; level >= 0; --level) {
            for (int iter = 0; iter < iterations[level]; ++iter) {
                float A[36], b[6], residual[2];
                be.icp_step(Rcurr->m, tcurr->v, vmaps_curr[level], nmaps_curr[level], Rprev_inv.m, tprev.v, intr.level(level),
                            vmaps_g_prev[level], nmaps_g_prev[level], cfg.rows >> level, cfg.cols >> level, distThres, angleThres,
                            A, b, residual);
                trace.insert(trace.end(), A, A + 36); trace.insert(trace.end(), b, b + 6); trace.insert(trace.end(), residual, residual + 2);
                ++icp_iters_done;
                double dA[36], db[6];
                for (int k = 0; k < 36; ++k) dA[k] = A[k];
                for (int k = 0; k < 6; ++k) db[k] = b[k];
                solveAndUpdate(dA, db, resultRt, Rprev, tprev, Rcurr, tcurr);
            }
        }
    }

    void populateRGBDData(const uint16_t* depth, const unsigned char* image, float** destDepths, unsigned char** destImages)  // RGBDOdometry.cpp:140-158
    {
        const int rows = cfg.rows, cols = cfg.cols;
        be.short_depth_to_metres(depth, destDepths[0], rows, cols, (int)(6.0 * 1000));
        for (int i = 0; i + 1 < LEVELS; ++i) be.pyrdown_gauss_f(destDepths[i], destDepths[i+1], rows >> i, cols >> i);
        be.bgr_to_intensity(image, destImages[0], rows, cols);
        for (int i = 0; i + 1 < LEVELS; ++i) be.pyrdown_uchar_gauss(destImages[i], destImages[i+1], rows >> i, cols >> i);
    }

    void rgbdOdometry(const Mat3f& Rprev, const Vec3f& tprev, Mat3f* Rcurr, Vec3f* tcurr)            // RGBDOdometry.cpp:165-393
    {
        const int rows = cfg.rows, cols = cfg.cols;
        Mat3f Rprev_inv = mat3_inverse_eigen(Rprev);
        populateRGBDData(depth_raw, rgb, nextDepth, nextImage);
        for (int i = 0; i < LEVELS; ++i) be.derivative_images(nextImage[i], nextdIdx[i], nextdIdy[i], rows >> i, cols >> i);
        double resultRt[16]; for (int k = 0; k < 16; ++k) resultRt[k] = (k % 5 == 0) ? 1.0 : 0.0;
        trace.clear(); icp_iters_done = 0;
        const float distThres = 0.10f, angleThres = sinf(20.f * 3.14159254f / 180.f);
        const double SOBEL_SCALE = 1.0 / std::pow(2.0, 3);
        const float MAX_DEPTH_DELTA = 0.07f;
        const int minimumGradientMagnitudes[4] = {12, 5, 3, 1};
        for (int i = LEVELS - 1; i >= 0; --i) {
            be.project_to_point_cloud(lastDepth[i], pointClouds[i], rows >> i, cols >> i, intrD, i);
            IntrD K = intrD.level(i);
            for (int j = 0; j < iterations[i]; ++j) {
                double Rt[16]; rigid4d_inverse(resultRt, Rt);                                        // :211
                // KRK_inv = K * R * K^-1 ; Kt = K * t   (:213-231), double then cast to float
                double R[9]; for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) R[a*3+b] = Rt[a*4+b];
                double Kd[9] = {K.fx, 0, K.cx, 0, K.fy, K.cy, 0, 0, 1};
                double Ki[9] = {1.0 / K.fx, 0, -K.cx / K.fx, 0, 1.0 / K.fy, -K.cy / K.fy, 0, 0, 1};
                double KR[9], KRKi[9];
                for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) { double s = 0; for (int k = 0; k < 3; ++k) s += Kd[a*3+k] * R[k*3+b]; KR[a*3+b] = s; }
                for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) { double s = 0; for (int k = 0; k < 3; ++k) s += KR[a*3+k] * Ki[k*3+b]; KRKi[a*3+b] = s; }
                float krkInv[9]; for (int n = 0; n < 9; ++n) krkInv[n] = (float)KRKi[n];
                float kt[3];
                for (int a = 0; a < 3; ++a) { double s = 0; for (int k = 0; k < 3; ++k) s += Kd[a*3+k] * Rt[k*4+3]; kt[a] = (float)s; }

                int sigma = 0, rgbSize = 0;
                float minScale = (float)(std::pow((double)minimumGradientMagnitudes[i], 2.0) / std::pow(SOBEL_SCALE, 2.0));
                be.rgb_residual(minScale, nextdIdx[i], nextdIdy[i], lastDepth[i], nextDepth[i], lastImage[i], nextImage[i],
                                corresImg[i], rows >> i, cols >> i, MAX_DEPTH_DELTA, kt, krkInv, &sigma, &rgbSize);
                // Q3: precedence makes this sqrt(rgbSize) unless sigma/rgbSize == 0 exactly.
                float sigmaVal = std::sqrt((float)sigma / rgbSize == 0 ? 1 : rgbSize);

                float A_icp[36] = {0}, b_icp[6] = {0}, residual[2] = {0, 0};
                if (cfg.odometry == 2)
                    be.icp_step(Rcurr->m, tcurr->v, vmaps_curr[i], nmaps_curr[i], Rprev_inv.m, tprev.v, intr.level(i),
                                vmaps_g_prev[i], nmaps_g_prev[i], rows >> i, cols >> i, distThres, angleThres, A_icp, b_icp, residual);
                float A_rgbd[36], b_rgbd[6];
                IntrF li = intr.level(i);
                be.rgb_step(corresImg[i], sigmaVal, pointClouds[i], li.fx, li.fy, nextdIdx[i], nextdIdy[i], (float)SOBEL_SCALE,
                            rows >> i, cols >> i, A_rgbd, b_rgbd);
                trace.insert(trace.end(), A_rgbd, A_rgbd + 36); trace.insert(trace.end(), b_rgbd, b_rgbd + 6);
                float cnt[2] = {(float)sigma, (float)rgbSize}; trace.insert(trace.end(), cnt, cnt + 2);
                ++icp_iters_done;
                double dA[36], db[6];
                if (cfg.odometry == 2) {
                    const double w = 10;                                                             // :316-321
                    for (int k = 0; k < 36; ++k) dA[k] = (double)A_rgbd[k] + w * w * (double)A_icp[k];
                    for (int k = 0; k < 6; ++k) db[k] = (double)b_rgbd[k] + w * (double)b_icp[k];
                } else {
                    for (int k = 0; k < 36; ++k) dA[k] = A_rgbd[k];
                    for (int k = 0; k < 6; ++k) db[k] = b_rgbd[k];
                }
                solveAndUpdate(dA, db, resultRt, Rprev, tprev, Rcurr, tcurr);
            }
        }
        for (int i = 0; i < LEVELS; ++i) { std::swap(lastDepth[i], nextDepth[i]); std::swap(lastImage[i], nextImage[i]); }   // :377-381
        float dx = tcurr->v[0] - tprev.v[0], dy = tcurr->v[1] - tprev.v[1], dz = tcurr->v[2] - tprev.v[2];
        if (std::sqrt(dx*dx + dy*dy + dz*dz) > 0.3) { *Rcurr = Rprev; *tcurr = tprev; }            // :383-387
    }
};

} // namespace kto
