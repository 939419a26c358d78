// deflate.h -- gzip file writers for the stages' .gz outputs.  Every writer writes the bytes gzopen(path, "w") + gzwrite + gzclose
// write with zlib's default level; GPU: deflate.cu (the pieces of deflate.cuh run in parallel), host: zlib itself.
#pragma once
#include <cstddef>
#include <string>

class GzFile {
public:
    virtual ~GzFile() {}
    // gzwrite: p is host memory, or device memory on the writer's device when on_device.  Any piece sizes give the same file.
    virtual void write(const void* p, size_t n, bool on_device) = 0;
    // gzclose: the last block, the trailer; the file is complete when this returns.  Throws on a write error.
    virtual void close() = 0;
};

// PGB200_GZ=gpu (default) or host.  The GPU writer is used only when its output equals the runtime zlib's on a probe text
// (gz_gpu_matches_zlib) and the device has room for its buffers; otherwise zlib writes and, under PGB200_VERBOSE, the stage says why.
// PGB200_GZ_CHUNK_MB sets the input per GPU round (default 32, at least 5).
GzFile* gz_open(const std::string& path, int device);
GzFile* gz_open_gpu(const std::string& path, int device, size_t chunk = 0);   // chunk 0: 32 MB of input per GPU round
GzFile* gz_open_host(const std::string& path);
bool gz_gpu_matches_zlib(int device);   // compares once per process; the result is kept
