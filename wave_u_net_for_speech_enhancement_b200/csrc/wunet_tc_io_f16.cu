// wunet_tc_io_f16.cu — the tensor-core inference kernels with an fp16 network input / output (wunet_tc_io.cuh).
#include <cuda_fp16.h>
#define WUNET_TC_IO __half
#define WUNET_TC_IO_NS io_f16
#include "wunet_tc_io.cuh"
