// Owning handles of the C-ABI (include/ltr_b200.h), shared by the device library and the host orchestrator.  Plain C++17.
#pragma once
#include <cstdint>
#include "../../include/ltr_b200.h"

namespace ltr {

// Owns one ltr_cloud / ltr_scanset / ltr_poses handle (-1: none) of a context and frees it when destroyed or reset, ignoring the
// status of the free.  Move-only; a moved-to owner takes the context along with the handle.
template <int (*Free)(ltr_ctx*, int32_t)>
class HandleOwner {
public:
    HandleOwner() = default;
    explicit HandleOwner(ltr_ctx* ctx, int32_t h = -1) : ctx_(ctx), h_(h) {}
    HandleOwner(HandleOwner&& o) noexcept : ctx_(o.ctx_), h_(o.release()) {}
    HandleOwner& operator=(HandleOwner&& o) noexcept { if (this != &o) { reset(); ctx_ = o.ctx_; h_ = o.release(); } return *this; }
    ~HandleOwner() { reset(); }
    int32_t get() const { return h_; }
    int32_t release() { const int32_t h = h_; h_ = -1; return h; }                  // the caller owns the handle from now on
    void reset(int32_t h = -1) { if (h_ >= 0 && h_ != h) Free(ctx_, h_); h_ = h; }   // frees the held handle unless it is h, takes h
private:
    ltr_ctx* ctx_ = nullptr;
    int32_t h_ = -1;
};
using CloudOwner = HandleOwner<ltr_cloud_free>;
using ScanSetOwner = HandleOwner<ltr_scanset_free>;
using PosesOwner = HandleOwner<ltr_poses_free>;

}  // namespace ltr
