// zb_host_stage.h -- staging helper behind the zb_host_* entry points: upload a host image into
// stream-ordered device scratch, run the device op, download the result and synchronise.  This is the
// literal drop-in for an Image(T) whose `data` lives in host memory (reference image.zig:97-102).
#pragma once
#include "zb_internal.h"

namespace zb {

struct HostStage {
    Scratch s_src, s_dst;
    zb_image dsrc{}, ddst{};
    cudaStream_t stream = nullptr;  // legacy default stream: ordered with everything, synchronous semantics

    // dst may have a different shape than src (resize / rotate).
    int begin(const zb_image* src, const zb_image* dst, int pixfmt) {
        if (exceeds_int_index(src, pixfmt) || exceeds_int_index(dst, pixfmt)) return ZB_ERR_UNSUPPORTED;   // before staging
        DeviceInfo di;
        int rc = device_info(&di);
        if (rc) return rc;
        const size_t pb = pixel_bytes(pixfmt);
        if ((rc = s_src.alloc((size_t)src->rows * src->cols * pb, stream))) return rc;
        if ((rc = s_dst.alloc((size_t)dst->rows * dst->cols * pb, stream))) return rc;
        dsrc = {s_src.p, src->rows, src->cols, src->cols};
        ddst = {s_dst.p, dst->rows, dst->cols, dst->cols};
        return zb_upload(src, &dsrc, pixfmt, (zb_stream)stream);
    }
    int finish(zb_image* dst, int pixfmt) {
        int rc = zb_download(&ddst, dst, pixfmt, (zb_stream)stream);
        if (rc) return rc;
        ZB_CUDA(cudaStreamSynchronize(stream));
        return ZB_OK;
    }
};

}  // namespace zb
