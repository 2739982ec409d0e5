// scanner/util/memory.h -- the buffer API op authors allocate outputs with (reference
// scanner/util/memory.h:39-67).  Same calls and ownership rules:
//   new_buffer / new_block_buffer / new_block_buffer_size / new_block_buffer_sizes allocate on a
//   DeviceHandle; a "block" is one allocation carved into N element buffers sharing one
//   refcount; add_buffer_ref(s) / delete_buffer adjust it by any pointer inside the block.
// This project's design (not the reference's first-fit pool under a global mutex, memory.cpp:164-267):
//   GPU blocks come from a per-device stream-ordered CUDA memory pool (cudaMallocAsync on the
//   device's pipeline stream, release threshold = unlimited so freed blocks are recycled without
//   touching the driver); CPU blocks are pinned host memory when a GPU is present so every
//   H2D/D2H is an async DMA.  Block lookup is an ordered interval map (one entry per block, not
//   per sub-pointer).
#pragma once
#include <cstddef>
#include <string>
#include <vector>

#include "scanner/util/common.h"

namespace scanner {

struct MemoryPoolConfig {
  bool pinned_cpu = true;        // CPU buffers are cudaHostAlloc'ed when CUDA is usable
  u64 gpu_release_threshold = ~0ull;
};

void init_memory_allocators(MemoryPoolConfig config, std::vector<i32> gpu_device_ids);
void destroy_memory_allocators();

u8* new_buffer_(DeviceHandle device, size_t size, const char* call_file, i32 call_line);
u8* new_block_buffer_(DeviceHandle device, size_t size, i32 refs, const char* call_file,
                      i32 call_line);
u8* new_block_buffer_sizes_(DeviceHandle device, const std::vector<size_t>& sizes,
                            const char* call_file, i32 call_line);
u8* new_block_buffer_size_(DeviceHandle device, size_t size, i32 copies, const char* call_file,
                           i32 call_line);

#define new_buffer(device__, size__) ::scanner::new_buffer_(device__, size__, __FILE__, __LINE__)
#define new_block_buffer(device__, size__, refs__) \
  ::scanner::new_block_buffer_(device__, size__, refs__, __FILE__, __LINE__)
#define new_block_buffer_sizes(device__, sizes__) \
  ::scanner::new_block_buffer_sizes_(device__, sizes__, __FILE__, __LINE__)
#define new_block_buffer_size(device__, size__, copies__) \
  ::scanner::new_block_buffer_size_(device__, size__, copies__, __FILE__, __LINE__)

void add_buffer_ref(DeviceHandle device, u8* buffer);
void add_buffer_refs(DeviceHandle device, u8* buffer, i32 refs);
void delete_buffer(DeviceHandle device, u8* buffer);

// Copies are asynchronous on the destination (or source) GPU's pipeline stream; memcpy_buffer
// returns after the copy is complete only when `sync` (default, matches the reference's
// blocking semantics, memory.cpp:863-891).
void memcpy_buffer(u8* dest_buffer, DeviceHandle dest_device, const u8* src_buffer,
                   DeviceHandle src_device, size_t size);
void memcpy_buffer_async(u8* dest_buffer, DeviceHandle dest_device, const u8* src_buffer,
                         DeviceHandle src_device, size_t size);
void memcpy_vec(std::vector<u8*>& dest_buffers, DeviceHandle dest_device,
                const std::vector<u8*>& src_buffers, DeviceHandle src_device,
                const std::vector<size_t>& sizes);
void copy_or_ref_buffers(std::vector<u8*>& dest_buffers, DeviceHandle dest_device,
                         const std::vector<u8*>& src_buffers, DeviceHandle src_device,
                         const std::vector<size_t>& sizes);

u64 current_memory_allocated(DeviceHandle device);
u64 max_memory_allocated(DeviceHandle device);

// --- additions to the reference's API -----------------------------------------------------------------------
// The CUDA stream all engine-issued work for GPU `id` is ordered on (cudaStream_t as void*).
// GPU kernels written against this API enqueue on it instead of the legacy default stream and
// do NOT synchronise before returning: the engine orders consumers on the same stream and
// synchronises once, when a result crosses to the host (SURVEY 8b "Sync convention").
void* device_stream(DeviceHandle device);
void sync_device(DeviceHandle device);
bool cuda_available();

}  // namespace scanner
