// jpeg_pipe.h -- device-resident JPEG re-encode pipe (see jpeg_pipe.cu)
#pragma once
#include <cstddef>
#include <cstdint>
#include <map>
#include <string>
#include <vector>
#include "../../include/b200_caesium.h"
#include "jpeg_host.h"

namespace b200 {
// the JPEG writer's options from the C ABI's parameters; copying the source's JFIF header is each caller's choice
inline JpegWriteOptions write_options(const b200_params *p)
{
    JpegWriteOptions wo; wo.progressive = p->jpeg_progressive != 0; wo.keep_metadata = p->keep_metadata != 0; wo.preserve_icc = p->jpeg_preserve_icc != 0;
    return wo;
}
struct JpegPipe;
JpegPipe *pipe_create(const uint8_t *const *in, const size_t *in_len, int n, const b200_params *p, int group_size, std::string &err);
// which: 0 whole path, 1 entropy decode only, 2 transform only, 3 entropy encode only (2 / 3 need a prior whole run)
bool pipe_run(JpegPipe *P, void *cuda_stream, int which, int *launches, std::string &err);
bool pipe_finish(JpegPipe *P, size_t *out_sizes, int *not_settled, int *enc_retries, std::string &err);
bool pipe_fetch(JpegPipe *P, int index, std::vector<uint8_t> &file, std::string &err);
bool pipe_kernel_times(JpegPipe *P, int iters, std::map<std::string, std::pair<double, int>> &out, std::string &err);
void pipe_destroy(JpegPipe *P);
int pipe_group_size(const JpegPipe *P);
int pipe_groups(const JpegPipe *P);
} // namespace b200
