// device_checks.h — argument checks of the entry points that read or write caller-owned device memory
// (cticp_odometry_register_device, cticp_odometry_write_points_device, cticp_trajectory_transform_device). They throw
// std::invalid_argument, which the C ABI reports as CTICP_ERR_INVALID_ARGUMENT, before anything is enqueued.
#pragma once
#include <cstdint>

#include "../../include/cticp.h"

namespace cticp {

// [p, p + bytes) must be device (or managed) memory of `device`, inside one allocation: a short buffer is an error here,
// not a fault in a kernel
void RequireDeviceRange(const void *p, uint64_t bytes, int device, const char *what);
// bytes spanned by n >= 1 records of `width` bytes every `stride` bytes
uint64_t SpanBytes(uint64_t n, uint64_t stride, uint64_t width, const char *what);
// the dtypes of a cticp_cloud_sink, and both of its fields inside the record (point_step)
void CheckSink(const cticp_cloud_sink &sink);
// the bytes a field of a sink record ends at: the later of the two fields
uint64_t SinkRecordWidth(const cticp_cloud_sink &sink);

}  // namespace cticp
