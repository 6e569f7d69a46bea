// wunet_tc_io_bf16.cu — the tensor-core inference kernels with a bf16 network input / output (wunet_tc_io.cuh).
#include <cuda_bf16.h>
#define WUNET_TC_IO __nv_bfloat16
#define WUNET_TC_IO_NS io_bf16
#include "wunet_tc_io.cuh"
