// Error plumbing shared by all translation units of libcis_b200.so: int status codes + a thread-local message,
// never throws, never exits (SURVEY.md section 8b "Errors").
#pragma once
#include <cuda_runtime.h>
int cis_set_error(int code, const char* msg);
int cis_set_cuda_error(cudaError_t e, const char* where);
int cis_check_launch(const char* where);
// streaming multiprocessors of the current device (132 on an H100 SXM); sizes one-wave and persistent grids
int cis_num_sms();
