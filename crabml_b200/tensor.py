"""CudaTensor: Python mirror of `impl Tensor for CudaTensor` (what the Rust crabml-cuda shim does),
over the C ABI.  Same method names / argument meaning / error behaviour as the reference trait
(crabml-core/src/tensor/api.rs:11-79) so parity tests read like the reference's backend tests
(crabml-wgpu/src/wgpu_tensor.rs:749-1099).  Metadata-only methods stay host-side (strider.rs)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi
from .capi import CudaError, TensorError, cc_view


class TensorStrider:
    """crabml-core/src/tensor/strider.rs:5-236 (host-side metadata; never crosses the ABI)."""

    def __init__(self, shape, strides=None):
        self.shape = [int(s) for s in shape]
        if strides is None:
            strides = [1]
            for i in range(len(self.shape) - 1):
                strides.append(strides[-1] * self.shape[len(self.shape) - i - 1])
            strides = strides[::-1]
        self.strides = [int(s) for s in strides]

    def clone(self): return TensorStrider(self.shape, self.strides)
    def dims(self): return len(self.shape)

    def len(self):
        n = 1
        for s in self.shape:
            n *= s
        return n

    def resize(self, new_shape):                                   # strider.rs:36-51
        if len(new_shape) != len(self.shape):
            raise TensorError(f"invalid new shape {new_shape} for a tensor of shape {self.shape}")
        return TensorStrider(new_shape, self.strides)

    def reshape(self, shape):                                      # strider.rs:143-160
        if not self.is_contiguous():
            raise TensorError("not contiguous")
        n = 1
        for s in shape:
            n *= s
        if n != self.len():
            raise TensorError(f"invalid shape {shape} for a tensor's origin shape {self.shape}")
        return TensorStrider(shape)

    def transpose(self, dims):                                     # strider.rs:162-180
        if len(dims) != len(self.shape):
            raise TensorError(f"invalid dims {dims} for a tensor of shape {self.shape}")
        return TensorStrider([self.shape[d] for d in dims], [self.strides[d] for d in dims])

    def is_contiguous(self):                                       # strider.rs:182-206
        if not self.strides:
            return True
        if self.strides[-1] != 1:
            return False
        last = 1
        for i in reversed(range(len(self.shape))):
            if last != self.strides[i]:
                return False
            last *= self.shape[i]
        return True


MEGA_NONE, MEGA_REGISTER, MEGA_RING = 0, 1, 2      # CudaTensorDevice.mega_variant(): MegaVariant (common.cuh)
MK_PROF_SLOTS = 10                                  # u64 stamps per phase of CudaTensorDevice.mega_profile() (common.cuh)


class CudaTensorDevice:
    """T::DeviceRef.  Options mirror CpuTensorDeviceOptions (cpu_device.rs:13-48)."""

    def __init__(self, ordinal=0, debug_named_tensors=False, lazy=False, exact_order=False):
        self.lib = capi.load_library()
        opts = capi.cc_device_options(ordinal, int(debug_named_tensors), int(lazy), int(exact_order), 0)
        h = C.c_void_p()
        rc = self.lib.cc_device_create(C.byref(opts), C.byref(h))
        if rc != capi.CC_OK:
            raise CudaError(self.lib.cc_last_error(None).decode())
        self.handle = h
        self.debug_named_tensors, self.lazy = debug_named_tensors, int(lazy)

    def check(self, rc):
        if rc == capi.CC_OK:
            return
        msg = self.lib.cc_last_error(self.handle).decode()
        if rc == capi.CC_ERR_TENSOR:
            raise TensorError(msg)
        raise CudaError(f"[{rc}] {msg}")

    def synchronize(self): self.check(self.lib.cc_device_synchronize(self.handle))

    # ---- sharded path: exchange window of this rank (comm.cu).  `exchange(bytes) -> [bytes of every rank]` is any
    # all-gather of small host blobs (torch.distributed.all_gather_object in bench.py / the tests) ----------------------------
    def init_comm(self, rank, world, exchange=None, transport="p2p"):
        handle = (C.c_uint8 * 64)()
        self.check(self.lib.cc_comm_create(self.handle, rank, world, handle))
        if world > 1 and exchange is None:
            raise CudaError("init_comm: an exchange function is required for world > 1")
        blobs = exchange(bytes(handle)) if world > 1 else [bytes(handle)]
        allh = (C.c_uint8 * (64 * world)).from_buffer_copy(b"".join(blobs))
        self.check(self.lib.cc_comm_connect(self.handle, allh))
        if transport == "nccl":
            uid = (C.c_uint8 * 128)()
            if rank == 0:
                self.check(self.lib.cc_comm_nccl_unique_id(self.handle, uid))
            uid0 = exchange(bytes(uid))[0] if world > 1 else bytes(uid)
            self.check(self.lib.cc_comm_init_nccl(self.handle, (C.c_uint8 * 128).from_buffer_copy(uid0)))
        elif transport != "p2p":
            raise CudaError(f"unknown transport {transport}")
        self.rank, self.world = rank, world

    def create_comm_local(self, rank, world):
        """first half of an in-process world (every rank is a device of THIS process): allocate the exchange window"""
        handle = (C.c_uint8 * 64)()
        self.check(self.lib.cc_comm_create(self.handle, rank, world, handle))
        self.rank, self.world = rank, world

    def connect_comm_local(self, devices):
        """second half: wire the windows of all ranks directly (devices[r] = the CudaTensorDevice of rank r)"""
        arr = (C.c_void_p * len(devices))(*[d.handle.value if hasattr(d.handle, "value") else d.handle for d in devices])
        self.check(self.lib.cc_comm_connect_local(self.handle, arr))

    def set_sm_limit(self, n): self.check(self.lib.cc_device_set_sm_limit(self.handle, int(n)))

    def timer_begin(self): self.check(self.lib.cc_bench_timer_begin(self.handle))

    def timer_end(self) -> float:
        ms = C.c_float(0)
        self.check(self.lib.cc_bench_timer_end(self.handle, C.byref(ms)))
        return float(ms.value)
    def launch_count(self): return int(self.lib.cc_device_launch_count(self.handle))
    def flush(self): self.check(self.lib.cc_device_flush(self.handle))

    def lazy_stats(self):
        a = (C.c_uint64 * 8)()
        if self.lib.cc_lazy_stats(self.handle, a) != capi.CC_OK:
            return None
        return {"flushes": a[0], "graph_replays": a[1], "graph_captures": a[2], "uncached": a[3],
                "host_us_record": a[4] / 1e3, "host_us_fuse": a[5] / 1e3, "host_us_submit": a[6] / 1e3, "ops": a[7]}

    def mega_variant(self) -> int:
        """MEGA_NONE none yet, MEGA_REGISTER mega_kernel (tables without a Q8_0 / Q4_0 matvec), MEGA_RING mega_ring_kernel (TMA-fed
        shared-memory ring)."""
        return int(self.lib.cc_lazy_mega_variant(self.handle))

    def mega_profile(self, max_phases=4096):
        """(stamps [phases + 1, MK_PROF_SLOTS] uint64, phase type codes) of the last captured persistent kernel; needs a lazy device
        created with CRABML_MEGA_PROF=1.  A type code is 16 * type (0 NORMQ, 1 MATVEC, 2 ATTN, 3 ROWS, 4 REDUCE, 5 GATHER, 6 ARGMAX,
        7 SAMPLE), plus for a MATVEC phase its matrix count + 4 * epilogue + 1024 * (k >> 10)."""
        cap = MK_PROF_SLOTS * (max_phases + 1)
        ts, ty, n = np.zeros(cap, np.uint64), (C.c_int32 * cap)(), C.c_int32(0)
        self.check(self.lib.cc_lazy_mega_profile(self.handle, ts.ctypes.data_as(C.POINTER(C.c_uint64)), ty, cap, C.byref(n)))
        return ts[:(n.value + 1) * MK_PROF_SLOTS].reshape(n.value + 1, MK_PROF_SLOTS), tuple(ty[:n.value])

    def mega_phase_types(self):
        """the phase type codes of the last captured persistent kernel (mega_profile)"""
        return self.mega_profile()[1]

    def read_history(self, first, count):
        """ids [first, first + count) of the device's history (sample_to_slot / cc_argmax_to_slot with hist_index >= 0)"""
        out = np.empty(count, np.int64)
        self.check(self.lib.cc_read_history(self.handle, first, count, out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def dump_debug_tensor(self, name):                              # cpu_device.rs:96-98
        n = C.c_size_t(0)
        rc = self.lib.cc_dump_debug_tensor(self.handle, name.encode(), None, C.byref(n))
        if rc != capi.CC_OK:
            return None
        out = np.empty(n.value, np.float32)
        self.check(self.lib.cc_dump_debug_tensor(self.handle, name.encode(), out.ctypes.data_as(C.c_void_p), C.byref(n)))
        return out

    def close(self):
        if self.handle:
            self.lib.cc_device_destroy(self.handle)
            self.handle = None


class _Buf:
    """Arc<buffer>: releases the device storage when the last Python reference dies."""

    def __init__(self, device, handle):
        self.device, self.handle = device, handle

    def __del__(self):
        try:
            if self.handle and self.device.handle:
                self.device.lib.cc_tensor_release(self.handle)
        except Exception:
            pass


def _shape_arr(shape):
    return (C.c_int64 * len(shape))(*[int(s) for s in shape])


class CudaTensor:
    def __init__(self, buf: _Buf, strider: TensorStrider, device: CudaTensorDevice, name=None):
        self.buf, self._strider, self.device, self.name = buf, strider, device, name

    # -- plumbing ------------------------------------------------------------------------------
    def _view(self):
        v = cc_view()
        v.buf = self.buf.handle
        v.ndim = len(self._strider.shape)
        if v.ndim > capi.CC_MAX_DIMS:
            raise TensorError("too many dims")
        for i, (s, t) in enumerate(zip(self._strider.shape, self._strider.strides)):
            v.shape[i], v.strides[i] = s, t
        return v

    def _new(self, handle, shape):
        return CudaTensor(_Buf(self.device, handle), TensorStrider(shape), self.device)

    # -- constructors (api.rs:14-23) -----------------------------------------------------------------
    @classmethod
    def from_cpu(cls, buf, shape, dtype, device):
        raw = np.ascontiguousarray(buf).view(np.uint8).reshape(-1) if isinstance(buf, np.ndarray) else np.frombuffer(bytes(buf), np.uint8)
        h = C.c_void_p()
        device.check(device.lib.cc_tensor_from_cpu(device.handle, raw.ctypes.data_as(C.c_void_p), raw.size, _shape_arr(shape), len(shape), dtype, C.byref(h)))
        return cls(_Buf(device, h), TensorStrider(shape), device)

    @classmethod
    def new(cls, values, shape, device):
        """CpuTensor::new analogue for tests: an OWNED F32 tensor initialised from host values."""
        values = np.ascontiguousarray(values, np.float32).reshape(-1)
        n = 1
        for s in shape:
            n *= s
        if values.size != n:
            raise TensorError(f"invalid shape {shape} for data of length {values.size}")
        src = cls.from_cpu(values, [n], capi.F32, device)
        t = cls.alloc([n], capi.F32, device)
        t.copy_rows_from(src, [0])
        return t.reshape(list(shape))

    @classmethod
    def alloc(cls, shape, dtype, device):
        h = C.c_void_p()
        device.check(device.lib.cc_tensor_alloc(device.handle, _shape_arr(shape), len(shape), dtype, C.byref(h)))
        return cls(_Buf(device, h), TensorStrider(shape), device)

    @classmethod
    def synth(cls, shape, dtype, device, seed, tensor_id, scale):
        h = C.c_void_p()
        device.check(device.lib.cc_tensor_synth(device.handle, _shape_arr(shape), len(shape), dtype, seed, tensor_id, scale, C.byref(h)))
        return cls(_Buf(device, h), TensorStrider(shape), device)

    @classmethod
    def synth_slice(cls, shape, dtype, device, seed, tensor_id, scale, row0, nrows, col0, ncols):
        """rows [row0, +nrows) x columns [col0, +ncols) of the tensor `synth` would generate (sharded path)."""
        h = C.c_void_p()
        device.check(device.lib.cc_tensor_synth_slice(device.handle, _shape_arr(shape), len(shape), dtype, seed, tensor_id, scale,
                                                      row0, nrows, col0, ncols, C.byref(h)))
        return cls(_Buf(device, h), TensorStrider([nrows, ncols]), device)

    # -- metadata (host side) ------------------------------------------------------------------------------
    def dtype(self): return int(self.device.lib.cc_tensor_dtype(self.buf.handle))
    def shape(self): return list(self._strider.shape)
    def strider(self): return self._strider
    def is_contiguous(self): return self._strider.is_contiguous()
    def _with(self, strider): return CudaTensor(self.buf, strider, self.device)

    def resize(self, axis, n):                                       # cpu_tensor.rs:167-197
        if axis >= len(self.shape()):
            raise TensorError(f"resize: axis {axis} is larger than the current shape {self.shape()}")
        new_shape = self.shape(); new_shape[axis] = n
        total = 1
        for s in new_shape:
            total *= s
        if total > self.device.lib.cc_tensor_capacity(self.buf.handle):
            raise TensorError(f"resize: new shape {new_shape} is larger than the current shape {self.shape()}")
        return self._with(self._strider.resize(new_shape))

    def with_strider(self, strider): return self._with(strider.clone())
    def reshape(self, shape): return self._with(self._strider.reshape(list(shape)))
    def transpose(self, dims): return self._with(self._strider.transpose(list(dims)))

    def with_name(self, name):                                        # cpu_tensor.rs:232-241
        self.name = name
        if self.device.debug_named_tensors:
            self.device.check(self.device.lib.cc_debug_tensor_tap(self.device.handle, name.encode(), C.byref(self._view())))
        return self

    # -- data movement -----------------------------------------------------------------------------------------
    def contiguous(self):
        h = C.c_void_p()
        self.device.check(self.device.lib.cc_contiguous(self.device.handle, C.byref(self._view()), C.byref(h)))
        if h.value == self.buf.handle.value:        # no-op path returned the same (retained) buffer
            self.device.lib.cc_tensor_release(h)
            return self
        return self._new(h, self.shape())

    def concatenate(self, rhs, axis):
        self.device.check(self.device.lib.cc_concatenate(self.device.handle, C.byref(self._view()), C.byref(rhs._view()), axis))
        new_shape = self.shape(); new_shape[axis] += rhs.shape()[axis]
        self._strider = self._strider.resize(new_shape)

    def copy_rows_from(self, src, rows):
        arr = (C.c_int64 * len(rows))(*[int(r) for r in rows])
        self.device.check(self.device.lib.cc_copy_rows_from(self.device.handle, C.byref(self._view()), C.byref(src._view()), arr, len(rows)))

    def export(self):
        out = np.empty(self._strider.len(), np.float32)
        self.device.check(self.device.lib.cc_tensor_export_f32(self.device.handle, C.byref(self._view()), out.ctypes.data_as(C.c_void_p), out.size))
        return out

    def to_vec(self):
        """test helper (cpu_tensor.rs:98-107): dense copy honouring strides."""
        return self.contiguous().export() if not self.is_contiguous() else self.export()

    def dup(self):
        h = C.c_void_p()
        self.device.check(self.device.lib.cc_tensor_dup(self.device.handle, C.byref(self._view()), C.byref(h)))
        return self._new(h, self.shape())

    # -- in-place ops (take self by value in Rust; here they return self) ----------------------------------------
    def _inplace(self, fn, *args):
        self.device.check(fn(self.device.handle, C.byref(self._view()), *args))
        return self

    def rope_inplace(self, mode, pos, rope_dims): return self._inplace(self.device.lib.cc_rope_inplace, mode, pos, rope_dims)
    def rms_norm_inplace(self, eps): return self._inplace(self.device.lib.cc_rms_norm_inplace, eps)
    def softmax_inplace(self, axis): return self._inplace(self.device.lib.cc_softmax_inplace, axis)
    def silu_inplace(self): return self._inplace(self.device.lib.cc_silu_inplace)
    def gelu_inplace(self): return self._inplace(self.device.lib.cc_gelu_inplace)
    def mul_inplace(self, rhs): return self._inplace(self.device.lib.cc_mul_inplace, C.byref(rhs._view()))
    def add_inplace(self, rhs): return self._inplace(self.device.lib.cc_add_inplace, C.byref(rhs._view()))
    def scale_inplace(self, rhs): return self._inplace(self.device.lib.cc_scale_inplace, float(rhs))

    # -- exchange step of the sharded path (crabml_cuda.h; not part of the reference's trait) ------------------
    def all_reduce_sum_inplace(self): return self._inplace(self.device.lib.cc_all_reduce_sum_inplace)

    def all_gather_from(self, piece):
        self.device.check(self.device.lib.cc_all_gather(self.device.handle, C.byref(self._view()), C.byref(piece._view())))
        return self

    # -- hot path ----------------------------------------------------------------------------------------------------
    def matmul_vec(self, x):
        h = C.c_void_p()
        self.device.check(self.device.lib.cc_matmul_vec(self.device.handle, C.byref(self._view()), C.byref(x._view()), C.byref(h)))
        m = self.shape()[0]
        return self._new(h, [m] if len(x.shape()) == 1 else [x.shape()[0], m])

    def batch_matmul(self, b):
        h = C.c_void_p()
        self.device.check(self.device.lib.cc_batch_matmul(self.device.handle, C.byref(self._view()), C.byref(b._view()), C.byref(h)))
        return self._new(h, [self.shape()[0], self.shape()[1], b.shape()[2]])

    # -- sampling on the device (crabml_cuda.h; not part of the reference's trait) ------------------------------------
    def sample_to_slot(self, temperature, topp, seed, coin_index, slot=0, hist_index=-1):
        """Llama2Sampler::sample (sampler.rs:27-107) of these logits into device slot `slot` (and history[hist_index] when >= 0);
        temperature 0 is the argmax.  Read the id back with the device's history (cc_read_history)."""
        self.device.check(self.device.lib.cc_sample_to_slot(self.device.handle, C.byref(self._view()), float(temperature), float(topp),
                                                            int(seed) & (2**64 - 1), int(coin_index), int(slot), int(hist_index)))
        return self

    # -- test hooks -----------------------------------------------------------------------------------------------------
    def quantize_activation(self, act_type, nbytes):
        out = np.empty(nbytes, np.uint8)
        self.device.check(self.device.lib.cc_test_quantize_activation(self.device.handle, C.byref(self._view()), act_type, out.ctypes.data_as(C.c_void_p), nbytes))
        return out

    def export_blocks(self, nbytes):
        out = np.empty(nbytes, np.uint8)
        self.device.check(self.device.lib.cc_test_export_blocks(self.device.handle, self.buf.handle, out.ctypes.data_as(C.c_void_p), nbytes))
        return out
