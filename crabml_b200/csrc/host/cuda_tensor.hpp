// cuda_tensor.hpp -- C++ mirror of `impl Tensor for CudaTensor` (what the Rust crabml-cuda crate would be),
// written against the C ABI only (include/crabml_cuda.h).  Same method names, ownership conventions and
// error behaviour as the reference trait (crabml-core/src/tensor/api.rs:11-79):
//   * "in-place" ops consume the tensor and hand it back (Rust: self by value -> Result<Self>),
//   * matmul_vec / batch_matmul / dup return a NEW tensor, concatenate / copy_rows_from mutate,
//   * clones share storage (refcounted cc_buf, like Arc<wgpu::Buffer> in crabml-wgpu/src/wgpu_tensor.rs:20-28),
//   * reshape / transpose / with_strider / resize are metadata-only (tensor/strider.rs) and never cross the ABI,
//   * errors surface as TensorError (ErrorKind::TensorError, error.rs:24-25) carrying cc_last_error().
#pragma once

#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../../include/crabml_cuda.h"

namespace crabml {

struct TensorError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// crabml-core/src/tensor/strider.rs:5-236
class TensorStrider {
public:
    TensorStrider() = default;
    explicit TensorStrider(std::vector<int64_t> shape) : shape_(std::move(shape)) {     // strider.rs:12-15,216-224
        strides_.assign(shape_.size(), 1);
        for (int i = (int)shape_.size() - 2; i >= 0; i--) strides_[i] = strides_[i + 1] * shape_[i + 1];
    }
    TensorStrider(std::vector<int64_t> shape, std::vector<int64_t> strides) : shape_(std::move(shape)), strides_(std::move(strides)) {}

    const std::vector<int64_t>& shape() const { return shape_; }
    const std::vector<int64_t>& strides() const { return strides_; }
    size_t dims() const { return shape_.size(); }
    int64_t len() const {
        int64_t n = 1;
        for (auto s : shape_) n *= s;
        return n;
    }
    TensorStrider resize(const std::vector<int64_t>& new_shape) const {                 // strider.rs:36-51
        if (new_shape.size() != shape_.size()) throw TensorError("invalid new shape for resize");
        return TensorStrider(new_shape, strides_);
    }
    TensorStrider reshape(const std::vector<int64_t>& shape) const {                    // strider.rs:143-160
        if (!is_contiguous()) throw TensorError("not contiguous");
        int64_t n = 1;
        for (auto s : shape) n *= s;
        if (n != len()) throw TensorError("invalid shape for reshape");
        return TensorStrider(shape);
    }
    TensorStrider transpose(const std::vector<int>& dims) const {                       // strider.rs:162-180
        if (dims.size() != shape_.size()) throw TensorError("invalid dims for transpose");
        std::vector<int64_t> s, t;
        for (int d : dims) { s.push_back(shape_[d]); t.push_back(strides_[d]); }
        return TensorStrider(s, t);
    }
    bool is_contiguous() const {                                                        // strider.rs:182-206
        if (strides_.empty()) return true;
        if (strides_.back() != 1) return false;
        int64_t last = 1;
        for (int i = (int)shape_.size() - 1; i >= 0; i--) {
            if (last != strides_[i]) return false;
            last *= shape_[i];
        }
        return true;
    }

private:
    std::vector<int64_t> shape_, strides_;
};

class CudaTensor {
public:
    CudaTensor() = default;
    CudaTensor(cc_device* dev, cc_buf* buf, TensorStrider st) : dev_(dev), buf_(buf), strider_(std::move(st)) {}   // adopts one reference
    CudaTensor(const CudaTensor& o) : dev_(o.dev_), buf_(o.buf_), strider_(o.strider_) { if (buf_) cc_tensor_retain(buf_); }
    CudaTensor(CudaTensor&& o) noexcept : dev_(o.dev_), buf_(o.buf_), strider_(std::move(o.strider_)) { o.buf_ = nullptr; }
    CudaTensor& operator=(CudaTensor o) noexcept {
        std::swap(dev_, o.dev_); std::swap(buf_, o.buf_); std::swap(strider_, o.strider_);
        return *this;
    }
    ~CudaTensor() { if (buf_) cc_tensor_release(buf_); }

    static CudaTensor wrap(cc_device* dev, cc_buf* borrowed, const std::vector<int64_t>& shape) {   // weights owned elsewhere
        if (!borrowed) throw TensorError("wrap: null tensor");
        int64_t n = 1;
        for (int64_t d : shape) n *= d;
        // a weight handed over with the wrong shape (config / file mismatch) must be a TensorError here, not a silent misread
        if (n != cc_tensor_capacity(borrowed))
            throw TensorError("wrap: shape has " + std::to_string(n) + " elements, the tensor holds " + std::to_string(cc_tensor_capacity(borrowed)));
        cc_tensor_retain(borrowed);
        return CudaTensor(dev, borrowed, TensorStrider(shape));
    }
    static CudaTensor alloc(const std::vector<int64_t>& shape, int dtype, cc_device* dev) {        // api.rs:23
        cc_buf* b = nullptr;
        check(dev, cc_tensor_alloc(dev, shape.data(), (int)shape.size(), dtype, &b));
        return CudaTensor(dev, b, TensorStrider(shape));
    }

    // ---- metadata-only (host side) ------------------------------------------------------------------
    bool valid() const { return buf_ != nullptr; }
    int dtype() const { return cc_tensor_dtype(buf_); }
    const std::vector<int64_t>& shape() const { return strider_.shape(); }
    const TensorStrider& strider() const { return strider_; }
    CudaTensor resize(int axis, int64_t n) && {                                          // cpu_tensor.rs:167-197
        if (axis >= (int)shape().size()) throw TensorError("resize: axis out of range");
        std::vector<int64_t> ns = shape();
        ns[axis] = n;
        int64_t total = 1;
        for (auto s : ns) total *= s;
        if (total > cc_tensor_capacity(buf_)) throw TensorError("resize: new shape is larger than the storage");
        strider_ = strider_.resize(ns);
        return std::move(*this);
    }
    CudaTensor with_strider(TensorStrider st) && { strider_ = std::move(st); return std::move(*this); }
    CudaTensor reshape(const std::vector<int64_t>& s) && { strider_ = strider_.reshape(s); return std::move(*this); }
    CudaTensor transpose(const std::vector<int>& d) && { strider_ = strider_.transpose(d); return std::move(*this); }
    CudaTensor with_name(const std::string& name) && {                                   // cpu_tensor.rs:232-241
        cc_view v = view();
        check(dev_, cc_debug_tensor_tap(dev_, name.c_str(), &v));
        return std::move(*this);
    }

    // ---- data movement ------------------------------------------------------------------------------------
    CudaTensor contiguous() && {                                                          // api.rs:40
        cc_view v = view();
        cc_buf* b = nullptr;
        check(dev_, cc_contiguous(dev_, &v, &b));
        if (b == buf_) { cc_tensor_release(b); return std::move(*this); }
        return CudaTensor(dev_, b, TensorStrider(shape()));
    }
    void concatenate(const CudaTensor& rhs, int axis) {                                   // api.rs:46
        cc_view a = view(), r = rhs.view();
        check(dev_, cc_concatenate(dev_, &a, &r, axis));
        std::vector<int64_t> ns = shape();
        ns[axis] += rhs.shape()[axis];
        strider_ = strider_.resize(ns);
    }
    void copy_rows_from(const CudaTensor& src, const std::vector<int64_t>& rows) {        // api.rs:50
        cc_view d = view(), s = src.view();
        check(dev_, cc_copy_rows_from(dev_, &d, &s, rows.data(), (int)rows.size()));
    }
    // greedy decoding without a host round trip per token (extension of the C ABI, crabml_cuda.h)
    void copy_rows_from_slot(const CudaTensor& src, int slot) {
        cc_view d = view(), s = src.view();
        check(dev_, cc_copy_rows_from_slot(dev_, &d, &s, slot));
    }
    void argmax_to_slot(int slot, int64_t hist_index) const {
        cc_view v = view();
        check(dev_, cc_argmax_to_slot(dev_, &v, slot, hist_index));
    }
    void sample_to_slot(float temperature, float topp, uint64_t seed, int64_t coin_index, int slot, int64_t hist_index) const {
        cc_view v = view();
        check(dev_, cc_sample_to_slot(dev_, &v, temperature, topp, seed, coin_index, slot, hist_index));
    }
    void export_async(float* dst, size_t n) const {
        cc_view v = view();
        check(dev_, cc_tensor_export_f32_async(dev_, &v, dst, n));
    }
    void export_to(float* dst, size_t n) const {                                          // api.rs:52
        cc_view v = view();
        check(dev_, cc_tensor_export_f32(dev_, &v, dst, n));
    }
    CudaTensor dup() const {                                                              // api.rs:55
        cc_view v = view();
        cc_buf* b = nullptr;
        check(dev_, cc_tensor_dup(dev_, &v, &b));
        return CudaTensor(dev_, b, TensorStrider(shape()));
    }

    // ---- in-place ops: consume and return (api.rs:57-74) ---------------------------------------------------------
    CudaTensor rope_inplace(int mode, int64_t pos, int64_t rope_dims) && { cc_view v = view(); check(dev_, cc_rope_inplace(dev_, &v, mode, pos, rope_dims)); return std::move(*this); }
    CudaTensor rms_norm_inplace(float eps) && { cc_view v = view(); check(dev_, cc_rms_norm_inplace(dev_, &v, eps)); return std::move(*this); }
    CudaTensor softmax_inplace(int axis) && { cc_view v = view(); check(dev_, cc_softmax_inplace(dev_, &v, axis)); return std::move(*this); }
    CudaTensor silu_inplace() && { cc_view v = view(); check(dev_, cc_silu_inplace(dev_, &v)); return std::move(*this); }
    CudaTensor gelu_inplace() && { cc_view v = view(); check(dev_, cc_gelu_inplace(dev_, &v)); return std::move(*this); }
    CudaTensor mul_inplace(const CudaTensor& rhs) && { cc_view v = view(), r = rhs.view(); check(dev_, cc_mul_inplace(dev_, &v, &r)); return std::move(*this); }
    CudaTensor add_inplace(const CudaTensor& rhs) && { cc_view v = view(), r = rhs.view(); check(dev_, cc_add_inplace(dev_, &v, &r)); return std::move(*this); }
    CudaTensor scale_inplace(float s) && { cc_view v = view(); check(dev_, cc_scale_inplace(dev_, &v, s)); return std::move(*this); }

    // ---- exchange step of the sharded path (not in the reference's trait: it is single-device; crabml_cuda.h) ------------
    CudaTensor all_reduce_sum_inplace() && { cc_view v = view(); check(dev_, cc_all_reduce_sum_inplace(dev_, &v)); return std::move(*this); }
    void all_gather_from(const CudaTensor& slice) { cc_view d = view(), s = slice.view(); check(dev_, cc_all_gather(dev_, &d, &s)); }

    // ---- hot path (api.rs:76-78) -----------------------------------------------------------------------------------
    CudaTensor matmul_vec(const CudaTensor& x) const {
        cc_view w = view(), xv = x.view();
        cc_buf* b = nullptr;
        check(dev_, cc_matmul_vec(dev_, &w, &xv, &b));
        std::vector<int64_t> s = x.shape().size() == 1 ? std::vector<int64_t>{shape()[0]} : std::vector<int64_t>{x.shape()[0], shape()[0]};
        return CudaTensor(dev_, b, TensorStrider(s));
    }
    CudaTensor batch_matmul(const CudaTensor& y) const {
        cc_view a = view(), bv = y.view();
        cc_buf* b = nullptr;
        check(dev_, cc_batch_matmul(dev_, &a, &bv, &b));
        return CudaTensor(dev_, b, TensorStrider({shape()[0], shape()[1], y.shape()[2]}));
    }

    cc_view view() const {
        cc_view v;
        v.buf = buf_;
        v.ndim = (int32_t)strider_.dims();
        if (v.ndim > CC_MAX_DIMS) throw TensorError("too many dims");
        for (int i = 0; i < v.ndim; i++) { v.shape[i] = strider_.shape()[i]; v.strides[i] = strider_.strides()[i]; }
        return v;
    }
    static void check(cc_device* dev, int rc) {
        if (rc != CC_OK) throw TensorError(std::string(cc_last_error(dev)));
    }

private:
    cc_device* dev_ = nullptr;
    cc_buf* buf_ = nullptr;
    TensorStrider strider_;
};

}  // namespace crabml
