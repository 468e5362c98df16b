// ply.h — PLY files on one device: columns of strided scalars packed into binary_little_endian files, many files per
// launch, and the host reader of pose files. Semantics, quirks and refusals: include/cticp.h, "PLY files".
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "../../include/cticp.h"

namespace cticp {

// m files of device columns into device memory, ordered on `stream`, no host synchronisation
void PlyWriteDevice(int device, const cticp_ply_property *props, uint64_t n_props, uint64_t num_items,
                    const uint64_t *file_ends, uint64_t m, void *out, uint64_t capacity, uint64_t *file_offsets,
                    cudaStream_t stream);
// one file of host columns into host bytes through the device (synchronous); returns the file size
uint64_t PlyWrite(int device, const cticp_ply_property *props, uint64_t n_props, uint64_t num_items, void *out,
                  uint64_t capacity);
// host only
std::vector<cticp_pose> PlyReadPoses(const char *bytes, uint64_t n);

}  // namespace cticp
