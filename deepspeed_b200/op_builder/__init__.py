"""Op builders.

Two shared libraries hold every native component:

* ``libdsb200_cuda.so`` -- all sm_90a kernels + the symmetric-memory (VMM/NVLS) runtime.
* ``libdsb200_cpu.so``  -- host runtime: AVX-512/AVX2 optimizers, async file I/O engine,
  shared-memory collectives, ragged-batch host helpers.

The per-op builder classes mirror the reference names (``FusedAdamBuilder``, ``CPUAdamBuilder``,
``AsyncIOBuilder`` ... see reference ``op_builder/*.py``) so ``get_accelerator().create_op_builder``
and ``ds_report`` keep working; ``load()`` returns the Python binding module for that op.
"""
import importlib

from .builder import (ARCH_FLAGS, BuildError, CPUOpBuilder, CUDAOpBuilder, LIB_DIR, OpBuilder, cuda_home,  # noqa: F401
                      nvcc_path)


class CudaKernelsBuilder(CUDAOpBuilder):
    NAME = "dsb200_cuda"
    SOURCES = [
        "cuda/optim.cu",
        "cuda/transformer.cu",
        "cuda/quant.cu",
        "cuda/moe_ragged.cu",
        "cuda/misc.cu",
        "cuda/symm_coll.cu",
        "cuda/gemm_sm90.cu",
        "cuda/fp8_cast.cu",
        "cuda/attention.cu",
        "cuda/attn_sm90.cu",
        "cuda/attn_bias.cu",
        "cuda/moe_symm.cu",
        "cuda/wq_gemm.cu",
        "cuda/wq_tc_gemm.cu",
        "cuda/symm_mem.cpp",
    ]
    LINK_LIBS = ["-ldl", "-lpthread"]


class CpuRuntimeBuilder(CPUOpBuilder):
    NAME = "dsb200_cpu"
    SOURCES = [
        "cpu/cpu_optim.cpp",
        "cpu/aio.cpp",
        "cpu/shm_comm.cpp",
        "cpu/host_utils.cpp",
    ]
    LINK_LIBS = ["-lpthread", "-lrt"]


class _BindingBuilder:
    """Named builder whose ``load()`` imports the python binding for one op family."""
    NAME = ""
    BINDING = ""
    LIB = CudaKernelsBuilder

    def __init__(self):
        self.name = self.NAME

    def absolute_name(self):
        return self.BINDING

    def is_compatible(self, verbose=False):
        return self.LIB().is_compatible(verbose)

    def installed(self):
        return self.LIB().installed()

    def sources(self):
        return self.LIB().sources()

    def include_paths(self):
        return self.LIB().include_paths()

    def load(self, verbose=False):
        self.LIB().load(verbose)
        return importlib.import_module(self.BINDING)

    jit_load = load

    def builder(self):
        return self.LIB()


def _mk(cls_name, name, binding, lib=CudaKernelsBuilder):
    return type(cls_name, (_BindingBuilder, ), {"NAME": name, "BINDING": binding, "LIB": lib})


FusedAdamBuilder = _mk("FusedAdamBuilder", "fused_adam", "deepspeed_b200.ops.adam.fused_adam")
FusedLambBuilder = _mk("FusedLambBuilder", "fused_lamb", "deepspeed_b200.ops.lamb.fused_lamb")
FusedLionBuilder = _mk("FusedLionBuilder", "fused_lion", "deepspeed_b200.ops.lion.fused_lion")
CPUAdamBuilder = _mk("CPUAdamBuilder", "cpu_adam", "deepspeed_b200.ops.adam.cpu_adam", CpuRuntimeBuilder)
CPUAdagradBuilder = _mk("CPUAdagradBuilder", "cpu_adagrad", "deepspeed_b200.ops.adagrad.cpu_adagrad",
                        CpuRuntimeBuilder)
CPULionBuilder = _mk("CPULionBuilder", "cpu_lion", "deepspeed_b200.ops.lion.cpu_lion", CpuRuntimeBuilder)
QuantizerBuilder = _mk("QuantizerBuilder", "quantizer", "deepspeed_b200.ops.quantizer.quantizer")
FPQuantizerBuilder = _mk("FPQuantizerBuilder", "fp_quantizer", "deepspeed_b200.ops.fp_quantizer.quantize")


def _fpq_default_dtype():
    """Container dtype of the packed codes (reference op_builder/fp_quantizer.py:106)."""
    import torch
    return torch.uint8


def _fpq_range(q_bits=None):
    """Largest representable magnitude of the minifloat format with ``q_bits`` storage bits (reference :111)."""
    from deepspeed_b200.ops.fp_quantizer.quantize import _MANTISSA, _fmt_max
    assert q_bits in _MANTISSA, f"Please specify the right quantization range for the selected precision {q_bits}!"
    return _fmt_max(q_bits, _MANTISSA[q_bits])


FPQuantizerBuilder.get_default_quant_dtype = staticmethod(_fpq_default_dtype)
FPQuantizerBuilder.get_quant_range = staticmethod(_fpq_range)
TransformerBuilder = _mk("TransformerBuilder", "transformer", "deepspeed_b200.ops.transformer.transformer")
StochasticTransformerBuilder = _mk("StochasticTransformerBuilder", "stochastic_transformer",
                                   "deepspeed_b200.ops.transformer.transformer")
InferenceBuilder = _mk("InferenceBuilder", "transformer_inference", "deepspeed_b200.ops.transformer.inference")
InferenceCoreBuilder = _mk("InferenceCoreBuilder", "inference_core_ops", "deepspeed_b200.inference.v2.kernels")
RaggedOpsBuilder = _mk("RaggedOpsBuilder", "ragged_device_ops", "deepspeed_b200.inference.v2.kernels")
InferenceCutlassBuilder = _mk("InferenceCutlassBuilder", "cutlass_ops", "deepspeed_b200.inference.v2.kernels")
RaggedUtilsBuilder = _mk("RaggedUtilsBuilder", "ragged_ops", "deepspeed_b200.inference.v2.ragged.host",
                         CpuRuntimeBuilder)
AsyncIOBuilder = _mk("AsyncIOBuilder", "async_io", "deepspeed_b200.ops.aio", CpuRuntimeBuilder)
GDSBuilder = _mk("GDSBuilder", "gds", "deepspeed_b200.ops.gds", CpuRuntimeBuilder)
RandomLTDBuilder = _mk("RandomLTDBuilder", "random_ltd", "deepspeed_b200.ops.random_ltd.dropping_utils")
SparseAttnBuilder = _mk("SparseAttnBuilder", "sparse_attn", "deepspeed_b200.ops.sparse_attention")
SpatialInferenceBuilder = _mk("SpatialInferenceBuilder", "spatial_inference", "deepspeed_b200.ops.spatial")
EvoformerAttnBuilder = _mk("EvoformerAttnBuilder", "evoformer_attn", "deepspeed_b200.ops.deepspeed4science")
UtilsBuilder = _mk("UtilsBuilder", "utils", "deepspeed_b200.ops.flatten")
ShareMemCommBuilder = _mk("ShareMemCommBuilder", "deepspeed_shm_comm", "deepspeed_b200.comm.shm", CpuRuntimeBuilder)
SymmMemBuilder = _mk("SymmMemBuilder", "symm_mem", "deepspeed_b200.comm.symm")
GemmSm100Builder = _mk("GemmSm100Builder", "gemm_sm100", "deepspeed_b200.ops.gemm")

ALL_OPS = {
    cls.NAME: cls
    for cls in (FusedAdamBuilder, FusedLambBuilder, FusedLionBuilder, CPUAdamBuilder, CPUAdagradBuilder,
                CPULionBuilder, QuantizerBuilder, FPQuantizerBuilder, TransformerBuilder,
                StochasticTransformerBuilder, InferenceBuilder, InferenceCoreBuilder, RaggedOpsBuilder,
                InferenceCutlassBuilder, RaggedUtilsBuilder, AsyncIOBuilder, GDSBuilder, RandomLTDBuilder,
                SparseAttnBuilder, SpatialInferenceBuilder, EvoformerAttnBuilder, UtilsBuilder, ShareMemCommBuilder,
                SymmMemBuilder, GemmSm100Builder)
}


def build_all(verbose=True):
    """Compile both native libraries (used by ``__graft_entry__.build`` and ``setup.py``)."""
    out = []
    for b in (CudaKernelsBuilder(), CpuRuntimeBuilder()):
        out.append(b.build(verbose=verbose))
    return out


def get_default_compute_capabilities():
    return "9.0a"


# ---- per-op module paths of the reference (``op_builder/fused_adam.py`` ...) ------------------------------------------------
# The reference has one file per builder; here every builder is a two-line class over the same two libraries, so the module
# paths are registered virtually instead of stamping out 21 one-line files: ``from deepspeed_b200.op_builder.fused_adam import
# FusedAdamBuilder`` resolves to a module object created on the spot that exposes exactly that class.
_MODULE_OF = {
    "async_io": AsyncIOBuilder, "cpu_adagrad": CPUAdagradBuilder, "cpu_adam": CPUAdamBuilder, "cpu_lion": CPULionBuilder,
    "evoformer_attn": EvoformerAttnBuilder, "fp_quantizer": FPQuantizerBuilder, "fused_adam": FusedAdamBuilder,
    "fused_lamb": FusedLambBuilder, "fused_lion": FusedLionBuilder, "gds": GDSBuilder,
    "inference_core_ops": InferenceCoreBuilder, "inference_cutlass_builder": InferenceCutlassBuilder,
    "quantizer": QuantizerBuilder, "ragged_ops": RaggedOpsBuilder, "ragged_utils": RaggedUtilsBuilder,
    "random_ltd": RandomLTDBuilder, "sparse_attn": SparseAttnBuilder, "spatial_inference": SpatialInferenceBuilder,
    "stochastic_transformer": StochasticTransformerBuilder, "transformer": TransformerBuilder,
    "transformer_inference": InferenceBuilder,
}


def _register_builder_modules(package_name):
    import sys
    import types
    for mod, cls in _MODULE_OF.items():
        full = f"{package_name}.{mod}"
        if full in sys.modules:
            continue
        m = types.ModuleType(full, f"``{cls.__name__}`` (reference ``op_builder/{mod}.py``); see ``op_builder/__init__.py``.")
        setattr(m, cls.__name__, cls)
        m.__package__ = package_name
        sys.modules[full] = m
        setattr(sys.modules[package_name], mod, m)


_register_builder_modules(__name__)
