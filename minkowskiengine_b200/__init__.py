"""minkowskiengine_b200 — an H100-native (sm_90a) backend for the sparse-convolution
hot path of NVIDIA/MinkowskiEngine, behind the reference's own Python API.

    import minkowskiengine_b200 as ME
    x = ME.SparseTensor(features, coordinates, device="cuda")
    y = ME.MinkowskiConvolution(64, 128, kernel_size=3, stride=2, dimension=3).cuda()(x)

Scope (SURVEY.md §8): SparseTensor / CoordinateManager / kernel maps, MinkowskiConvolution,
MinkowskiConvolutionTranspose, MinkowskiChannelwiseConvolution (depthwise), local pooling and
unpooling (MinkowskiPoolingTranspose), global pooling, broadcast, batch and instance
normalisation, pruning, union and arithmetic between sparse tensors on different coordinate maps,
TensorField (point features quantised to voxels or splatted onto their corners, sliced back and
interpolated, and pooled per cloud or broadcast onto directly), dense-tensor interop (SparseTensor.dense, MinkowskiToDenseTensor, to_sparse,
to_sparse_all, dense_coordinates), COO sparse-times-dense products (spmm, spmm_average) and max
pooling over an explicit pair list, and the thin torch wrappers (cat / sum / mean / var, the stack containers,
MinkowskiToFeature) that MinkUNet, the ResNet classifiers and generative networks need.
CUDA tensors only; all device work runs in csrc/libmeb200.so (include/meb200.h).
"""
__version__ = "0.1.0"

from . import _lib
from .backend import (CoordinateMapKey, cuda_version, cudart_version, get_gpu_memory_info,
                      is_cuda_available)
from .enums import (BroadcastMode, ConvolutionMode, CoordinateMapType, CUDAKernelMapMode,
                    GPUMemoryAllocatorType, MinkowskiAlgorithm, PoolingMode, RegionType)
from .kernel_generator import (KernelGenerator, KernelRegion, convert_region_type,
                               get_kernel_volume)
from .sparse_tensor import (SparseTensor, SparseTensorOperationMode,
                            SparseTensorQuantizationMode, clear_global_coordinate_manager,
                            global_coordinate_manager, set_global_coordinate_manager,
                            set_sparse_tensor_operation_mode, sparse_tensor_operation_mode)
from .common import MinkowskiModuleBase, convert_to_int_list, convert_to_int_tensor
from .coordinate_manager import (CoordinateManager, CoordsManager, set_gpu_allocator,
                                 set_memory_manager_backend)
from .convolution import (MinkowskiConvolution, MinkowskiConvolutionFunction,
                          MinkowskiConvolutionTranspose, MinkowskiConvolutionTransposeFunction,
                          MinkowskiGenerativeConvolutionTranspose)
from .channelwise_convolution import (MinkowskiChannelwiseConvolution,
                                      MinkowskiChannelwiseConvolutionFunction)
from .pooling import (MinkowskiAvgPooling, MinkowskiDirectMaxPoolingFunction,
                      MinkowskiGlobalAvgPooling, MinkowskiGlobalMaxPooling,
                      MinkowskiGlobalPooling, MinkowskiGlobalPoolingFunction,
                      MinkowskiGlobalSumPooling, MinkowskiLocalPoolingFunction,
                      MinkowskiLocalPoolingTransposeFunction, MinkowskiMaxPooling,
                      MinkowskiPoolingTranspose, MinkowskiSumPooling)
from .broadcast import (MinkowskiBroadcast, MinkowskiBroadcastAddition,
                        MinkowskiBroadcastConcatenation, MinkowskiBroadcastFunction,
                        MinkowskiBroadcastMultiplication)
from .normalization import (MinkowskiBatchNorm, MinkowskiInstanceNorm,
                            MinkowskiInstanceNormFunction, MinkowskiSyncBatchNorm, fused_bn_relu)
from .convolution import fused_conv_bn_relu
from .backend import fp8_inference, fp8_training
from .fp8_calibration import Fp8Calibration
from .fp8_delayed import Fp8DelayedScaling
from .nonlinearity import *  # noqa: F401,F403
from .ops import (MinkowskiLinear, MinkowskiStackCat, MinkowskiStackMean, MinkowskiStackSum,
                  MinkowskiStackVar, MinkowskiToFeature, MinkowskiToSparseTensor, cat, mean, var)
from .ops import sum  # noqa: A004 -- ME.sum, the reference's name
from .tensor_field import TensorField
from .interpolation import MinkowskiInterpolation, MinkowskiInterpolationFunction
from .pruning import MinkowskiPruning, MinkowskiPruningFunction
from .union import MinkowskiUnion, MinkowskiUnionFunction
from .dense import (MinkowskiDenseToRowsFunction, MinkowskiToDenseFunction, MinkowskiToDenseTensor,
                    dense_coordinates, to_sparse, to_sparse_all)
from .sparse_matrix_functions import (MinkowskiSPMMAverageFunction, MinkowskiSPMMFunction, spmm,
                                      spmm_average)
from . import modules, utils  # noqa: F401
