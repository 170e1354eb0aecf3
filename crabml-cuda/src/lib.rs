//! CUDA (H100 / sm_90a) backend of crabml's `Tensor` trait.
//!
//! `CudaTensor` implements `crabml::tensor::Tensor` (crabml-core/src/tensor/api.rs:11-79) on top of the C ABI of
//! `libcrabml_cuda.so` (`include/crabml_cuda.h`): quantized GGUF blocks stay quantized on the device, the decode
//! hot path (`matmul_vec` on Q8_0 / Q4_0 / K-quant blocks) runs as hand-written CUDA kernels, and with
//! `CudaTensorDeviceOptions::with_lazy(2)` the ~1000 trait calls of one `Llama2Runner::forward` are recorded and
//! executed as ONE persistent kernel at the `export` that ends the forward pass.
//!
//! ```ignore
//! let device = CudaTensorDevice::new(CudaTensorDeviceOptions::new().with_lazy(2))?;
//! let model = GpuLlamaModel::<CudaTensor>::from_cpu(&model_cpu, device)?;   // needs integration/model_rs.diff
//! let mut runner = Llama2Runner::new(&model, conf.seq_len, false)?;
//! ```
mod device;
pub mod ffi;
mod tensor;

pub use device::CudaTensorDevice;
pub use device::CudaTensorDeviceOptions;
pub use device::CudaTensorDeviceRef;
pub use tensor::CudaTensor;
