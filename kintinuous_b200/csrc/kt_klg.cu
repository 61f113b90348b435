// kintinuous_b200 -- .klg log reader with the decode on the path to the device: the step BEFORE the hot path (SURVEY.md section 8 row f2).
//
// Replaces (reference):
//   RawLogReader::RawLogReader / readNext / hasMore            src/utils/RawLogReader.cpp:20-41, :52-133, RawLogReader.h
//   the upload + processFrame call of TrackerInterface::process src/backend/TrackerInterface.cpp:82-104
// File layout (RawLogReader.cpp:29, :54-66): int32 numFrames; per frame int64 timestamp, int32 depthSize, int32 imageSize, depthSize bytes
// (zlib stream of rows*cols u16, or the raw 2*rows*cols bytes), imageSize bytes (a JPEG, or the raw 3*rows*cols bytes, or nothing).
// The reference inflates and cvDecodeImage-s on the CPU into pageable buffers, then uploads with a blocking cudaMemcpy2D
// (containers/device_memory.cpp:258-267).  Here:
//   * depth is inflated straight into PINNED memory and copied to the device asynchronously;
//   * a JPEG image never exists on the host in decoded form: nvJPEG (a CUDA-toolkit library, like cuBLAS: plumbing, not the product)
//     decodes it on the device into the interleaved BGR bytes cvDecodeImage would have produced (the reference then labels them r,g,b,
//     RawLogReader.cpp:122 / -f flips them);
//   * two buffer sets alternate, so frame k+1 can be read and decoded while the tracker still works on frame k.
// zlib and nvJPEG are bound with dlopen when the first log is opened: the tracking library itself has no load-time dependency on them.
// Decoders differ in IDCT rounding / chroma upsampling: the depth is exact, a decoded JPEG agrees with libjpeg's to a few grey levels
// (tolerance stated in tests/test_gpu_klg.py).
#include "kt_ops.h"
#include "../../include/kintinuous_b200.h"
#include <nvjpeg.h>
#include <dlfcn.h>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

using namespace kt;

namespace {

typedef int (*uncompress_fn)(unsigned char*, unsigned long*, const unsigned char*, unsigned long);
typedef nvjpegStatus_t (*nvjpegCreateSimple_fn)(nvjpegHandle_t*);
typedef nvjpegStatus_t (*nvjpegDestroy_fn)(nvjpegHandle_t);
typedef nvjpegStatus_t (*nvjpegJpegStateCreate_fn)(nvjpegHandle_t, nvjpegJpegState_t*);
typedef nvjpegStatus_t (*nvjpegJpegStateDestroy_fn)(nvjpegJpegState_t);
typedef nvjpegStatus_t (*nvjpegGetImageInfo_fn)(nvjpegHandle_t, const unsigned char*, size_t, int*, nvjpegChromaSubsampling_t*, int*, int*);
typedef nvjpegStatus_t (*nvjpegDecode_fn)(nvjpegHandle_t, nvjpegJpegState_t, const unsigned char*, size_t, nvjpegOutputFormat_t, nvjpegImage_t*, cudaStream_t);

struct Codecs {
    void* zlib; void* nvj; bool tried;
    uncompress_fn uncompress;
    nvjpegCreateSimple_fn create; nvjpegDestroy_fn destroy; nvjpegJpegStateCreate_fn state_create; nvjpegJpegStateDestroy_fn state_destroy;
    nvjpegGetImageInfo_fn info; nvjpegDecode_fn decode;
};
Codecs g_codecs;

int load_codecs()
{
    Codecs& c = g_codecs;
    if (!c.tried) {
        c.tried = true;
        c.zlib = dlopen("libz.so.1", RTLD_NOW | RTLD_LOCAL);
        if (c.zlib) c.uncompress = (uncompress_fn)dlsym(c.zlib, "uncompress");
        c.nvj = dlopen("libnvjpeg.so.12", RTLD_NOW | RTLD_LOCAL);
        if (!c.nvj) c.nvj = dlopen("libnvjpeg.so", RTLD_NOW | RTLD_LOCAL);
        if (c.nvj) {
            c.create = (nvjpegCreateSimple_fn)dlsym(c.nvj, "nvjpegCreateSimple"); c.destroy = (nvjpegDestroy_fn)dlsym(c.nvj, "nvjpegDestroy");
            c.state_create = (nvjpegJpegStateCreate_fn)dlsym(c.nvj, "nvjpegJpegStateCreate"); c.state_destroy = (nvjpegJpegStateDestroy_fn)dlsym(c.nvj, "nvjpegJpegStateDestroy");
            c.info = (nvjpegGetImageInfo_fn)dlsym(c.nvj, "nvjpegGetImageInfo"); c.decode = (nvjpegDecode_fn)dlsym(c.nvj, "nvjpegDecode");
        }
    }
    return 0;
}

__global__ void __launch_bounds__(256) swap_rb_kernel(uint8_t* __restrict__ rgb, int n)          // cv::cvtColor(rgb, rgb, CV_RGB2BGR), RawLogReader.cpp:117-125
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t a = rgb[3 * i], b = rgb[3 * i + 2];
    rgb[3 * i] = b; rgb[3 * i + 2] = a;
}

} // namespace

struct kt_klg {
    FILE* fp; int rows, cols, device; int32_t num_frames; int current; int flip_colors;
    size_t P;
    std::vector<unsigned char> comp_depth, comp_image;       // compressedDepth / compressedImage (RawLogReader.cpp:31-32)
    Allocations mem;
    uint16_t* depth_pinned[2]; uint8_t* image_pinned[2];      // decompressionBuffer / raw image, pinned
    uint16_t* depth_dev[2]; uint8_t* rgb_dev[2];
    cudaStream_t stream; cudaEvent_t done[2];
    nvjpegHandle_t nvj; nvjpegJpegState_t nvj_state; bool nvj_ready;
    int set;                                                  // buffer set of the frame handed out last
    kt_klg_frame last;
    ~kt_klg()
    {
        cudaSetDevice(device);
        if (stream) cudaStreamSynchronize(stream);
        if (nvj_ready) { g_codecs.state_destroy(nvj_state); g_codecs.destroy(nvj); }
        if (fp) fclose(fp);
    }
};

extern "C" {

int kt_klg_open(const char* path, int rows, int cols, int device, kt_klg** out)
{
    if (!path || !out || rows <= 0 || cols <= 0) { set_error("kt_klg_open: bad argument"); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(device));
    load_codecs();
    FILE* fp = fopen(path, "rb");
    if (!fp) { set_error("kt_klg_open: cannot open %s", path); return KT_ERR_INVALID; }
    int32_t n = 0;
    if (fread(&n, sizeof(int32_t), 1, fp) != 1 || n < 0) { fclose(fp); set_error("kt_klg_open: %s has no frame count", path); return KT_ERR_INVALID; }
    std::unique_ptr<kt_klg> k(new kt_klg());
    k->fp = fp; k->rows = rows; k->cols = cols; k->device = device; k->num_frames = n; k->current = 0; k->flip_colors = 0; k->set = 1;
    k->P = (size_t)rows * cols;
    k->comp_depth.resize(k->P * 2); k->comp_image.resize(k->P * 3);
    const char* W = "kt_klg_open buffers";
    int r;
    for (int i = 0; i < 2; ++i)
        if ((r = k->mem.pinned(&k->depth_pinned[i], k->P, W)) || (r = k->mem.pinned(&k->image_pinned[i], k->P * 3, W)) ||
            (r = k->mem.device(&k->depth_dev[i], k->P, W)) || (r = k->mem.device(&k->rgb_dev[i], k->P * 3, W)) ||
            (r = k->mem.event(&k->done[i], cudaEventDisableTiming, W))) return r;
    if ((r = k->mem.stream(&k->stream, W))) return r;
    memset(&k->last, 0, sizeof(k->last));
    *out = k.release();
    return KT_OK;
}

int kt_klg_close(kt_klg* k)
{
    delete k;
    return KT_OK;
}

int kt_klg_num_frames(kt_klg* k) { return k ? k->num_frames : 0; }
int kt_klg_has_more(kt_klg* k) { return k && k->current + 1 < k->num_frames ? 1 : 0; }          // LogReader::hasMore: currentFrame + 1 < numFrames (RawLogReader.h)
int kt_klg_set_flip_colors(kt_klg* k, int flip) { if (!k) return KT_ERR_INVALID; k->flip_colors = flip != 0; return KT_OK; }

// RawLogReader::readNext (:52-133).  On return the frame's depth and image are on their way to the device on the reader's stream;
// kt_klg_wait (or kt_klg_track_next) orders a consumer behind them.
int kt_klg_read_next(kt_klg* k, kt_klg_frame* out)
{
    if (!k) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(k->device));
    const int s = k->set ^ 1;
    // the buffer set we are about to fill was handed out two frames ago; its previous transfers are long done, but be exact about it
    KT_CUDA(cudaEventSynchronize(k->done[s]));
    int64_t ts = 0; int32_t dsz = 0, isz = 0;
    if (fread(&ts, sizeof(int64_t), 1, k->fp) != 1 || fread(&dsz, sizeof(int32_t), 1, k->fp) != 1 || fread(&isz, sizeof(int32_t), 1, k->fp) != 1) {
        set_error("kt_klg_read_next: end of file at frame %d of %d", k->current, k->num_frames); return KT_ERR_STATE;
    }
    if (dsz < 0 || isz < 0 || (size_t)dsz > k->P * 2 || (size_t)isz > k->P * 3) { set_error("kt_klg_read_next: frame %d has sizes %d / %d", k->current, dsz, isz); return KT_ERR_INVALID; }
    if (dsz && fread(k->comp_depth.data(), (size_t)dsz, 1, k->fp) != 1) { set_error("kt_klg_read_next: truncated depth"); return KT_ERR_STATE; }
    if (isz && fread(k->comp_image.data(), (size_t)isz, 1, k->fp) != 1) { set_error("kt_klg_read_next: truncated image"); return KT_ERR_STATE; }
    int compressed = 0;
    // ---- image (:71-96) ----
    if ((size_t)isz == k->P * 3) {
        memcpy(k->image_pinned[s], k->comp_image.data(), k->P * 3);
        KT_CUDA(cudaMemcpyAsync(k->rgb_dev[s], k->image_pinned[s], k->P * 3, cudaMemcpyHostToDevice, k->stream));
    } else if (isz > 0) {
        compressed = 1;
        Codecs& c = g_codecs;
        if (!c.nvj || !c.create || !c.decode || !c.info) { set_error("kt_klg_read_next: frame %d holds a JPEG and libnvjpeg.so.12 could not be loaded", k->current); return KT_ERR_INVALID; }
        if (!k->nvj_ready) {
            if (c.create(&k->nvj) != NVJPEG_STATUS_SUCCESS || c.state_create(k->nvj, &k->nvj_state) != NVJPEG_STATUS_SUCCESS) { set_error("nvjpegCreateSimple failed"); return KT_ERR_CUDA; }
            k->nvj_ready = true;
        }
        int comps = 0, w[NVJPEG_MAX_COMPONENT], h[NVJPEG_MAX_COMPONENT]; nvjpegChromaSubsampling_t sub;
        if (c.info(k->nvj, k->comp_image.data(), (size_t)isz, &comps, &sub, w, h) != NVJPEG_STATUS_SUCCESS || w[0] != k->cols || h[0] != k->rows) {
            set_error("kt_klg_read_next: frame %d: JPEG is not %d x %d", k->current, k->cols, k->rows); return KT_ERR_INVALID;
        }
        nvjpegImage_t img; memset(&img, 0, sizeof(img));
        img.channel[0] = k->rgb_dev[s]; img.pitch[0] = (size_t)k->cols * 3;
        // cvDecodeImage yields interleaved B,G,R bytes
        const nvjpegStatus_t st = c.decode(k->nvj, k->nvj_state, k->comp_image.data(), (size_t)isz, NVJPEG_OUTPUT_BGRI, &img, k->stream);
        if (st != NVJPEG_STATUS_SUCCESS) { set_error("nvjpegDecode failed on frame %d (status %d)", k->current, (int)st); return KT_ERR_CUDA; }
    } else {
        KT_CUDA(cudaMemsetAsync(k->rgb_dev[s], 0, k->P * 3, k->stream));
    }
    // ---- depth (:98-122) ----
    if ((size_t)dsz == k->P * 2) {
        if (compressed) { set_error("kt_klg_read_next: frame %d: raw depth with a compressed image", k->current); return KT_ERR_INVALID; }   // assert(!isCompressed)
        memcpy(k->depth_pinned[s], k->comp_depth.data(), k->P * 2);
    } else if (dsz > 0) {
        if (!g_codecs.uncompress) { set_error("kt_klg_read_next: frame %d holds zlib depth and libz.so.1 could not be loaded", k->current); return KT_ERR_INVALID; }
        unsigned long len = (unsigned long)(k->P * 2);
        const int zr = g_codecs.uncompress((unsigned char*)k->depth_pinned[s], &len, k->comp_depth.data(), (unsigned long)dsz);
        if (zr != 0 || len != k->P * 2) { set_error("kt_klg_read_next: frame %d: zlib returned %d, %lu bytes", k->current, zr, len); return KT_ERR_INVALID; }
        compressed = 1;
    } else {
        memset(k->depth_pinned[s], 0, k->P * 2);
        compressed = 0;
    }
    KT_CUDA(cudaMemcpyAsync(k->depth_dev[s], k->depth_pinned[s], k->P * 2, cudaMemcpyHostToDevice, k->stream));
    if (k->flip_colors) { swap_rb_kernel<<<div_up((int)k->P, 256), 256, 0, k->stream>>>(k->rgb_dev[s], (int)k->P); KT_LAUNCH_CHECK(); }
    KT_CUDA(cudaEventRecord(k->done[s], k->stream));
    k->set = s;
    ++k->current;
    kt_klg_frame f;
    f.timestamp = ts; f.depth_size = dsz; f.image_size = isz; f.is_compressed = compressed; f.frame = k->current;
    f.depth_dev = k->depth_dev[s]; f.rgb_dev = k->rgb_dev[s]; f.depth_host = k->depth_pinned[s];
    f.compressed_depth = k->comp_depth.data(); f.compressed_image = k->comp_image.data();
    k->last = f;
    if (out) *out = f;
    return KT_OK;
}

int kt_klg_wait(kt_klg* k)
{
    if (!k) return KT_ERR_INVALID;
    KT_CUDA(cudaEventSynchronize(k->done[k->set]));
    return KT_OK;
}

// The body of TrackerInterface::process (:82-104): next frame of the log -> device -> processFrame.
int kt_klg_track_next(kt_klg* k, kt_ctx* ctx, kt_pose* out)
{
    if (!k || !ctx) return KT_ERR_INVALID;
    kt_klg_frame f;
    int r = kt_klg_read_next(k, &f); if (r) return r;
    if ((r = kt_klg_wait(k))) return r;
    return kt_process_frame_device(ctx, f.depth_dev, f.rgb_dev, (uint64_t)f.timestamp, out);
}

}
