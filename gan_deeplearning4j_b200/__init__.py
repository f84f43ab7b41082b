"""gan_deeplearning4j_b200 -- host-side mirror of the DL4J ComputationGraph / Layer API for the GAN training
step of hamaadshah/gan_deeplearning4j, executing in libb200gan.so (hand-written sm_90a CUDA, include/b200gan.h).
No CPU fallback: compute entry points raise B200GanError when the CUDA library or an H100 is missing."""
from ._lib import B200GanError, LIB_PATH, PROTOTYPES, load  # noqa: F401
from .engine import BF16, FP32, EPI_ACTBWD, EPI_BNBWD, EPI_PLAIN, EPI_STATS, Context, Gan, Net, comm_unique_id, test_bn, test_conv, test_conv_ex, test_dropout, test_dropout_kind, test_ew, test_loss, test_pool  # noqa: F401
from . import data, models, parallel, serializer  # noqa: F401
