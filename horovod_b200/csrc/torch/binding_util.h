// Host-side helpers shared by the translation units of the PyTorch binding (binding.cc, optim_binding.cc,
// sync_bn_binding.cc, moe_binding.cc): the dtype map, the device and stream of a launch, the launch-error check, the
// argument checks several entry points make, and the last-CTA ticket cache.  Every entry point checks all of its
// arguments before it stages, allocates or launches anything.
#pragma once
#include <torch/extension.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime.h>
#include <map>
#include <mutex>
#include "../common/common.h"

namespace py = pybind11;

namespace hvd {

inline DataType MapDtype(at::ScalarType t) {
  switch (t) {
    case at::kByte: return DataType::UINT8;
    case at::kChar: return DataType::INT8;
    case at::kShort: return DataType::INT16;
    case at::kInt: return DataType::INT32;
    case at::kLong: return DataType::INT64;
    case at::kHalf: return DataType::FLOAT16;
    case at::kBFloat16: return DataType::BFLOAT16;
    case at::kFloat: return DataType::FLOAT32;
    case at::kDouble: return DataType::FLOAT64;
    case at::kBool: return DataType::BOOL;
    default: throw std::invalid_argument(std::string("Horovod: unsupported tensor dtype ") + c10::toString(t));
  }
}

// The device guard and the current CUDA stream of `t`'s device, for a launch on that stream.
struct OnDevice {
  explicit OnDevice(const at::Tensor& t) : guard(t.device()), stream(c10::cuda::getCurrentCUDAStream(t.get_device())) {}
  c10::cuda::CUDAGuard guard;
  cudaStream_t stream;
};

inline void CheckLaunch(const char* op, cudaError_t e) {
  TORCH_CHECK(e == cudaSuccess, op, " launch failed: ", cudaGetErrorString(e));
}

// what[i] of a list that one launch reads: a dense CUDA tensor on first's device with first's dtype (first = what[0]).
inline void CheckEntry(const char* op, const char* what, size_t i, const at::Tensor& t, const at::Tensor& first) {
  TORCH_CHECK(t.is_cuda() && t.is_non_overlapping_and_dense(), op, ": ", what, "[", i, "] must be a dense CUDA tensor");
  TORCH_CHECK(t.device() == first.device(), op, ": ", what, "[", i, "] is on ", t.device(), ", ", what, "[0] on ",
              first.device());
  TORCH_CHECK(t.scalar_type() == first.scalar_type(), op, ": ", what, "[", i, "] is ", t.scalar_type(), ", ", what,
              "[0] is ", first.scalar_type(), " (one dtype per call)");
}

// what[i], which the kernels address with the element indices of like_what[i] (`like`): like's device, sizes and
// strides, and the dtype `dtype`.  A mismatch would otherwise become an out-of-bounds access or silent garbage.
inline void CheckLike(const char* op, const char* what, size_t i, const at::Tensor& t, at::ScalarType dtype,
                      const char* like_what, const at::Tensor& like) {
  TORCH_CHECK(t.device() == like.device(), op, ": ", what, "[", i, "] is on ", t.device(), ", ", like_what, "[", i, "] on ",
              like.device());
  TORCH_CHECK(t.scalar_type() == dtype, op, ": ", what, "[", i, "] is ", t.scalar_type(), ", expected ", dtype);
  TORCH_CHECK(t.sizes() == like.sizes(), op, ": ", what, "[", i, "] has size ", t.sizes(), ", ", like_what, "[", i,
              "] has ", like.sizes());
  TORCH_CHECK(t.strides() == like.strides(), op, ": ", what, "[", i, "] has strides ", t.strides(), ", ", like_what, "[",
              i, "] has ", like.strides());
}

// A contiguous tensor of n elements (at_least: n or more) of one of `dtypes` on the CUDA device `dev`.
inline void CheckVector(const char* op, const char* what, const at::Tensor& t, const at::Device& dev,
                        std::initializer_list<at::ScalarType> dtypes, int64_t n, bool at_least = false) {
  TORCH_CHECK(t.device() == dev, op, ": ", what, " must be on ", dev, ", got ", t.device());
  TORCH_CHECK(t.is_contiguous() && (at_least ? t.numel() >= n : t.numel() == n), op, ": ", what, " must be contiguous with ",
              at_least ? "at least " : "", n, " elements, got sizes ", t.sizes());
  TORCH_CHECK(std::find(dtypes.begin(), dtypes.end(), t.scalar_type()) != dtypes.end(), op, ": ", what, " must be ",
              c10::Join(" or ", dtypes), ", got ", t.scalar_type());
}

// An optional one-element T scalar that the kernels read on the CUDA device `dev`: its address, nullptr when absent.
template <typename T>
const T* DeviceScalar(const char* op, const char* what, const c10::optional<at::Tensor>& t, const at::Device& dev) {
  if (!t.has_value() || !t->defined()) return nullptr;
  const at::ScalarType dtype = c10::CppTypeToScalarType<T>::value;
  TORCH_CHECK(t->device() == dev && t->scalar_type() == dtype && t->numel() == 1, op, ": ", what, " must be a one-element ",
              dtype, " tensor on ", dev, ", got ", t->numel(), " ", t->scalar_type(), " elements on ", t->device());
  return t->data_ptr<T>();
}

// The last-CTA tickets of the kernels that elect one (gradient statistics, SyncBatchNorm, MoE routing): at least n
// zeroed counters per (device, stream), which every launch leaves zeroed.  Launches on one stream run one after another
// and share them; launches on different streams may overlap and must not.  They come from torch's allocator and are
// zeroed on the stream, so a stream first seen while it is being captured (hvd.GraphedStep captures on a stream of its
// own) gets its array from the graph's pool, zeroed by the graph.  Arrays are kept for the life of the process: a
// captured graph may still refer to them.
inline unsigned* StreamTickets(int device, cudaStream_t s, int64_t n) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, at::Tensor> tickets;
  static std::vector<at::Tensor> outgrown;
  std::lock_guard<std::mutex> l(mu);
  at::Tensor& t = tickets[{device, s}];
  if (!t.defined() || t.numel() < n) {
    if (t.defined()) outgrown.push_back(t);
    t = at::zeros({std::max<int64_t>(n, 1024)}, at::TensorOptions().dtype(at::kInt).device(at::kCUDA, device));
  }
  return reinterpret_cast<unsigned*>(t.data_ptr<int>());
}

// The entry points of each subsystem, registered into the module by PYBIND11_MODULE in binding.cc.
void DefOptim(py::module_& m);
void DefSyncBn(py::module_& m);
void DefMoe(py::module_& m);

}  // namespace hvd
