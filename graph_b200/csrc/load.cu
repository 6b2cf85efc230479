// load.cu — graph files streamed between the file and device memory: Graph500 and text edge lists parsed into
// device edge arrays, and binary CSR files read into and written from the device CSR arrays.
//
// load_graph opens the file once.  Below LOAD_DEVICE_MIN_BYTES the host decoders of io.cu read it whole in
// pageable memory and their result is uploaded.  Larger files go through a ring of pinned buffers
// (PinnedRing): chunk k of the file travels through buffer k % ring.  On a load, one reader thread per buffer
// preads the chunks that map to it (ChunkReader), a copy stream moves each chunk to the device slot's staging
// buffer (DeviceStaging), and kernels on a work stream decode it.  On a save the copy stream fills the buffers
// from device memory and the host writes them out.  Ordering rules:
//   - a pinned buffer is refilled only after the copy out of it has completed (its `copied` event);
//   - a device staging buffer is overwritten or reallocated only after the kernels that read it have completed
//     (its `parsed` event);
//   - on every exit, errors included, the copy stream is drained before any buffer it writes into is freed;
//   - the ring's buffers go back to PinnedRingCache for the next load or save and are not freed; one that finds
//     the cache in use allocates its own ring and frees it.
//
//   Graph500: records never straddle a chunk (chunks are a multiple of 48 bytes = 4 records), m = len / 12 is
//   known up front, and k_load_graph500 decodes 4 records per thread with three 128-bit loads.
//   Text: a chunk ends at its last '\n'; the bytes after it are carried into the next chunk.  The edge index
//   of a line is the number of '\n' before it, so edges come out in file order: k_load_count_lines counts
//   the '\n' of each 4 KB tile, a CUB scan turns the counts into tile bases, and k_load_parse_text finds the
//   line starts of a tile from 128-bit loads (a block scan ranks them) and parses one line per start
//   (edgelist_scan.h).  m is unknown until the end, so the edge arrays grow; values the device parser
//   declines are listed (file offset, edge index) and re-parsed on the host with gb::parse_line.  Both build
//   the graph from the device arrays (graph_from_device_arrays), so it is the one the host readers followed by
//   gb_[di]graph_from_edges_u32 give.
//   Binary: the host preads the headers (bin_parse gives the section table) and every chunk is cut against the
//   table.  u32 sections without values go from the pinned buffer straight into their CSR array; a chunk that
//   meets another section is staged with the bytes of the element it cuts carried in front, and k_bin_split
//   narrows the ids and splits the records.
//   Writer: the file is pieces of host and device memory; chunk k + 1 is copied from the device into the ring
//   while chunk k is written with pwrite to a temporary file, which is then renamed over the destination.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <condition_variable>
#include <cstdlib>
#include <memory>
#include <thread>

#include <cub/cub.cuh>

#include "binary_format.h"
#include "common.cuh"
#include "edgelist_line.h"
#include "edgelist_scan.h"

namespace gb {

constexpr unsigned LOAD_BLOCK = 256;                    // threads per CTA of the text kernels
constexpr unsigned LOAD_TILE = LOAD_BLOCK * 16;         // bytes per CTA: one 128-bit load per thread
constexpr uint64_t LOAD_DEFAULT_CHUNK = 64ull << 20;    // bytes per pinned buffer
constexpr uint64_t LOAD_MIN_CHUNK = 64ull << 10;        // smallest buffer chosen for a small file
constexpr uint64_t LOAD_CARRY_RESERVE = 4096;           // pinned bytes in front of a chunk for the carried line
constexpr unsigned LOAD_RING = 4;                       // pinned buffers (and reader threads)

struct LoadCounters {
  unsigned int declined;  // text values re-parsed on the host
  unsigned int wide;      // an id above 32 bits was seen
};

// bit j set = byte pos + j is '\n' and lies before len
__device__ __forceinline__ uint32_t newline_mask(uint4 v, uint64_t pos, uint64_t len) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t m = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t eq = __vcmpeq4(w[k], 0x0A0A0A0Au);  // 0xFF in every byte that is '\n'
#pragma unroll
    for (int b = 0; b < 4; ++b) m |= ((eq >> (8 * b + 7)) & 1u) << (4 * k + b);
  }
  if (pos >= len) return 0;
  if (len - pos < 16) m &= (1u << (len - pos)) - 1u;
  return m;
}

__global__ void __launch_bounds__(LOAD_BLOCK) k_load_count_lines(const uint4* __restrict__ buf, uint64_t len,
                                                                 uint32_t* __restrict__ counts) {
  using Reduce = cub::BlockReduce<uint32_t, LOAD_BLOCK>;
  __shared__ typename Reduce::TempStorage tmp;
  const uint64_t i = (uint64_t)blockIdx.x * LOAD_BLOCK + threadIdx.x;
  const uint32_t c = __popc(newline_mask(buf[i], 16 * i, len));
  const uint32_t total = Reduce(tmp).Sum(c);
  if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// incl[t] = '\n' in tiles 0..t of the chunk; edge_base = edges of the earlier chunks; file_off = file
// position of buf[0].  Lines start at 0 and after every '\n' that is not the chunk's last byte.
__global__ void __launch_bounds__(LOAD_BLOCK) k_load_parse_text(const uint4* __restrict__ buf, uint64_t len,
                                                                const uint32_t* __restrict__ incl,
                                                                uint64_t edge_base, uint64_t file_off,
                                                                int want_value, uint32_t* __restrict__ src,
                                                                uint32_t* __restrict__ dst, float* __restrict__ w,
                                                                LoadCounters* __restrict__ ctr,
                                                                uint64_t* __restrict__ declined_off,
                                                                uint32_t* __restrict__ declined_edge) {
  using Scan = cub::BlockScan<uint32_t, LOAD_BLOCK>;
  __shared__ typename Scan::TempStorage tmp;
  const uint64_t i = (uint64_t)blockIdx.x * LOAD_BLOCK + threadIdx.x;
  const uint64_t pos = 16 * i;
  uint32_t m = newline_mask(buf[i], pos, len);
  uint32_t before;
  Scan(tmp).ExclusiveSum((uint32_t)__popc(m), before);
  uint64_t e = edge_base + (blockIdx.x ? incl[blockIdx.x - 1] : 0u) + before;  // '\n' before this segment
  const char* text = reinterpret_cast<const char*>(buf);
  bool wide = false;
  auto parse = [&](uint64_t start, uint64_t edge) {
    ScannedLine sl;
    scan_line(text, start, len, want_value != 0, &sl);
    wide |= (sl.src | sl.dst) > 0xFFFFFFFFull;
    src[edge] = (uint32_t)sl.src;
    dst[edge] = (uint32_t)sl.dst;
    if (want_value) {
      w[edge] = sl.value;
      if (sl.declined) {
        const unsigned int k = atomicAdd(&ctr->declined, 1u);
        declined_off[k] = file_off + start;
        declined_edge[k] = (uint32_t)edge;
      }
    }
  };
  if (i == 0 && len > 0) parse(0, edge_base);
  while (m) {
    const int j = __ffs(m) - 1;
    m &= m - 1;
    ++e;  // this '\n' is before the line it ends
    if (pos + j + 1 < len) parse(pos + j + 1, e);
  }
  if (__syncthreads_or(wide) && threadIdx.x == 0) atomicOr(&ctr->wide, 1u);
}

// PackedEdge{v0_low, v1_low, high} (graph500.rs:111-127): 4 records = 48 bytes = three 128-bit loads per
// thread; edge_base is a multiple of 4, so the src / dst stores are 128-bit too.
__global__ void k_load_graph500(const uint4* __restrict__ buf, uint64_t nrec, uint64_t edge_base,
                                uint32_t* __restrict__ src, uint32_t* __restrict__ dst,
                                LoadCounters* __restrict__ ctr) {
  uint32_t high = 0;
  const uint64_t groups = (nrec + 3) / 4;
  for (uint64_t g = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; g < groups;
       g += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t r0 = 4 * g;
    if (r0 + 4 <= nrec) {
      const uint4 a = buf[3 * g], b = buf[3 * g + 1], c = buf[3 * g + 2];
      *reinterpret_cast<uint4*>(src + edge_base + r0) = make_uint4(a.x, a.w, b.z, c.y);
      *reinterpret_cast<uint4*>(dst + edge_base + r0) = make_uint4(a.y, b.x, b.w, c.z);
      high |= a.z | b.y | c.x | c.w;
    } else {
      const uint32_t* words = reinterpret_cast<const uint32_t*>(buf);
      for (uint64_t r = r0; r < nrec; ++r) {
        src[edge_base + r] = words[3 * r];
        dst[edge_base + r] = words[3 * r + 1];
        high |= words[3 * r + 2];
      }
    }
  }
  if (__any_sync(0xFFFFFFFFu, high != 0) && (threadIdx.x & 31) == 0) atomicOr(&ctr->wide, 1u);
}

__global__ void k_load_patch(const uint32_t* __restrict__ edge, const float* __restrict__ val, uint64_t count,
                             float* __restrict__ w) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    w[edge[i]] = val[i];
}

// 32 bits at an unaligned byte position of a device buffer whose base is 4-byte aligned (may read 4 bytes past)
__device__ __forceinline__ uint32_t load_u32_at(const uint8_t* base, uint64_t pos) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(base + (pos & ~3ull));
  const uint32_t shift = (uint32_t)(pos & 3) * 8;
  return shift ? __funnelshift_r(w[0], w[1], shift) : w[0];
}

// Binary files: elements [first, first + count) of a section staged in buf, whose byte 0 is file byte buf_off.
// Element e starts at file byte sec + e * stride with an id of id_bytes (u64 ids are narrowed; a high word
// that is not 0 sets *wide), followed by an f32 value that goes to w[e] when w is not NULL.
__global__ void k_bin_split(const uint8_t* __restrict__ buf, uint64_t buf_off, uint64_t sec, uint32_t stride,
                            uint32_t id_bytes, uint64_t first, uint64_t count, uint32_t* __restrict__ ids,
                            float* __restrict__ w, unsigned int* __restrict__ wide) {
  bool big = false;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t e = first + i;
    const uint64_t pos = sec + e * stride - buf_off;
    ids[e] = load_u32_at(buf, pos);
    if (id_bytes == 8) big |= load_u32_at(buf, pos + 4) != 0;
    if (w) w[e] = __uint_as_float(load_u32_at(buf, pos + id_bytes));
  }
  if (__any_sync(0xFFFFFFFFu, big) && (threadIdx.x & 31) == 0) atomicOr(wide, 1u);
}

// Target<u32, f32> records (8 bytes, #[repr(C)]) from the SoA arrays, for the writer
__global__ void k_bin_interleave(const uint32_t* __restrict__ tgt, const float* __restrict__ w, uint64_t count,
                                 uint2* __restrict__ out) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    out[i] = make_uint2(tgt[i], __float_as_uint(w[i]));
}

// ---- host side ---------------------------------------------------------------------------------------
static uint64_t env_chunk_bytes() {
  const char* s = std::getenv("GB_LOAD_CHUNK_BYTES");
  if (!s || !*s) return 0;
  const unsigned long long v = std::strtoull(s, nullptr, 10);
  return v;
}

static bool pread_all(int fd, char* dst, uint64_t bytes, uint64_t off) {
  while (bytes) {
    const ssize_t r = ::pread(fd, dst, bytes, (off_t)off);
    if (r < 0 && errno == EINTR) continue;
    if (r <= 0) return false;
    dst += r;
    off += (uint64_t)r;
    bytes -= (uint64_t)r;
  }
  return true;
}

// a file open for reading, its size, and the path its errors name
struct InputFile {
  const char* path = nullptr;
  int fd = -1;
  uint64_t bytes = 0;
  ~InputFile() {
    if (fd >= 0) ::close(fd);
  }
  gb_status open(const char* p) {
    path = p;
    fd = ::open(p, O_RDONLY | O_CLOEXEC);
    if (fd < 0) return fail(GB_ERR_INVALID, "cannot open %s: %s", p, std::strerror(errno));
    struct stat st {};
    if (::fstat(fd, &st) != 0 || !S_ISREG(st.st_mode)) return fail(GB_ERR_INVALID, "%s is not a regular file", p);
    bytes = (uint64_t)st.st_size;
    return GB_OK;
  }
  // the whole file in host memory (not zero-filled first), for the host decoders
  gb_status read_all(std::unique_ptr<char[]>* out) const {
    out->reset(new (std::nothrow) char[bytes ? bytes : 1]);
    if (!*out) return fail(GB_ERR_OOM, "host allocation of %llu bytes failed", (unsigned long long)bytes);
    if (bytes && !pread_all(fd, out->get(), bytes, 0)) return fail(GB_ERR_INVALID, "reading %s failed", path);
    return GB_OK;
  }
};

struct PinnedBuf {
  char* p = nullptr;
  ~PinnedBuf() {
    if (p) cudaFreeHost(p);
  }
};

// Pinning host memory costs about as much as reading it from the page cache, so the ring is kept for the
// next load (at most LOAD_RING buffers of one default chunk each).
struct PinnedRingCache {
  std::mutex mu;
  bool busy = false;
  std::vector<char*> bufs;
  uint64_t bytes = 0;  // of each buffer
};
static PinnedRingCache& pinned_ring_cache() {
  static PinnedRingCache* c = new PinnedRingCache();  // never destroyed: no CUDA call at process exit
  return *c;
}

// The pinned buffers a file streams through, LOAD_CARRY_RESERVE bytes then one chunk each, and per buffer the
// event recorded behind the last copy out of it (into it, for the writer).  Chunk k is bytes
// [k * chunk, min((k + 1) * chunk, read_end)) of the file and goes through buffer k % ring.
struct PinnedRing {
  uint64_t chunk = 0, read_end = 0, nchunks = 0;
  unsigned ring = 0;
  std::vector<PinnedBuf> host;      // [ring]
  bool cached = false;              // host[] belongs to the pinned ring cache
  std::vector<cudaEvent_t> copied;  // [ring]

  // the geometry for streaming `bytes`: chunks of GB_LOAD_CHUNK_BYTES, else of a quarter of the file within
  // [LOAD_MIN_CHUNK, LOAD_DEFAULT_CHUNK] so that a small file keeps every buffer busy; then rounded down to
  // whole `unit`s (the Graph500 loader's 4-record groups)
  void plan(uint64_t bytes, uint64_t unit = 1) {
    chunk = env_chunk_bytes();
    if (chunk == 0) {
      const uint64_t quarter = (bytes / LOAD_RING + 4095) & ~(uint64_t)4095;
      chunk = std::min(LOAD_DEFAULT_CHUNK, std::max(LOAD_MIN_CHUNK, quarter));
    }
    chunk = std::max<uint64_t>(chunk, 16);  // >= the largest binary element: it spans at most two chunks
    chunk = std::max(unit, chunk / unit * unit);
    read_end = bytes;
    nchunks = (bytes + chunk - 1) / chunk;
    ring = (unsigned)std::min<uint64_t>(LOAD_RING, std::max<uint64_t>(nchunks, 1));
  }
  uint64_t chunk_bytes(uint64_t k) const { return std::min(chunk, read_end - k * chunk); }
  char* data(unsigned r) { return host[r].p + LOAD_CARRY_RESERVE; }

  // the buffers (the cached ones when the cache is free and they are large enough) and their events
  gb_status acquire() {
    host.resize(ring);
    copied.assign(ring, nullptr);
    const uint64_t bytes = LOAD_CARRY_RESERVE + chunk;
    PinnedRingCache& pc = pinned_ring_cache();
    {
      std::lock_guard<std::mutex> lock(pc.mu);
      if (!pc.busy && bytes <= LOAD_CARRY_RESERVE + LOAD_DEFAULT_CHUNK) {
        pc.busy = cached = true;
        if (pc.bytes < bytes || pc.bufs.size() < ring) {
          for (char* p : pc.bufs) cudaFreeHost(p);
          pc.bufs.clear();
          pc.bytes = std::max(pc.bytes, bytes);
          for (unsigned r = 0; r < ring; ++r) {
            char* p = nullptr;
            if (cudaHostAlloc(reinterpret_cast<void**>(&p), pc.bytes, cudaHostAllocDefault) != cudaSuccess) {
              cudaGetLastError();
              for (char* q : pc.bufs) cudaFreeHost(q);
              pc.bufs.clear();
              pc.bytes = 0;
              pc.busy = cached = false;
              break;
            }
            pc.bufs.push_back(p);
          }
        }
        for (unsigned r = 0; cached && r < ring; ++r) host[r].p = pc.bufs[r];
      }
    }
    for (unsigned r = 0; r < ring; ++r) {
      if (!cached) GB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&host[r].p), bytes, cudaHostAllocDefault));
      GB_CUDA(cudaEventCreateWithFlags(&copied[r], cudaEventDisableTiming));
    }
    return GB_OK;
  }

  ~PinnedRing() {
    for (cudaEvent_t e : copied) {
      if (e) cudaEventSynchronize(e), cudaEventDestroy(e);  // no copy may still use a buffer
    }
    if (cached) {
      for (auto& h : host) h.p = nullptr;  // back to the cache, not freed
      PinnedRingCache& pc = pinned_ring_cache();
      std::lock_guard<std::mutex> lock(pc.mu);
      pc.busy = false;
    }
  }
};

struct StreamPair {
  cudaStream_t copy = nullptr, work = nullptr;
  ~StreamPair() {
    if (copy) cudaStreamSynchronize(copy), cudaStreamDestroy(copy);
    if (work) cudaStreamSynchronize(work), cudaStreamDestroy(work);
  }
};

// The reader threads over a ring: thread r preads chunks r, r + R, ... into buffer r, each after the consumer
// has released the buffer for it and the copy out of it has completed.
struct ChunkReader : PinnedRing {
  int fd = -1, device = 0;
  std::vector<uint64_t> filled;        // [ring]: chunk index + 1 the buffer holds (0: none yet)
  std::vector<uint64_t> released_for;  // [ring]: the buffer may be filled with this chunk
  std::vector<std::thread> threads;
  std::mutex mu;
  std::condition_variable cv;
  bool stop = false, failed = false;
  std::string error;

  ChunkReader(int fd, int device) : fd(fd), device(device) {}
  gb_status start() {
    GB_TRY(acquire());
    filled.assign(ring, 0);
    for (unsigned r = 0; r < ring; ++r) released_for.push_back(r);
    for (unsigned r = 0; r < ring; ++r) threads.emplace_back([this, r] { run(r); });
    return GB_OK;
  }

  void run(unsigned r) {
    cudaSetDevice(device);
    for (uint64_t k = r; k < nchunks; k += ring) {
      {
        std::unique_lock<std::mutex> lock(mu);
        cv.wait(lock, [&] { return stop || released_for[r] == k; });
        if (stop) return;
      }
      const bool ok = cudaEventSynchronize(copied[r]) == cudaSuccess &&
                      pread_all(fd, data(r), chunk_bytes(k), k * chunk);
      std::lock_guard<std::mutex> lock(mu);
      if (!ok) {
        failed = true;
        error = "reading the file failed";
        cv.notify_all();
        return;
      }
      filled[r] = k + 1;
      cv.notify_all();
    }
  }

  gb_status wait_filled(uint64_t k) {
    const unsigned r = (unsigned)(k % ring);
    std::unique_lock<std::mutex> lock(mu);
    cv.wait(lock, [&] { return failed || filled[r] == k + 1; });
    if (failed) return fail(GB_ERR_INVALID, "%s", error.c_str());
    return GB_OK;
  }

  // every copy out of chunk k's buffer is issued on sp.copy: the buffer is refilled once they complete, and
  // sp.work waits for them
  gb_status release(uint64_t k, const StreamPair& sp) {
    const unsigned r = (unsigned)(k % ring);
    GB_CUDA(cudaEventRecord(copied[r], sp.copy));
    {
      std::lock_guard<std::mutex> lock(mu);
      released_for[r] = k + ring;
    }
    cv.notify_all();
    GB_CUDA(cudaStreamWaitEvent(sp.work, copied[r], 0));
    return GB_OK;
  }

  ~ChunkReader() {  // then ~PinnedRing waits for the copies out of the buffers
    {
      std::lock_guard<std::mutex> lock(mu);
      stop = true;
    }
    cv.notify_all();
    for (auto& t : threads) t.join();
  }
};

// The device side of a streamed load: per ring slot a staging buffer and the event recorded behind the kernels
// that read it.  Chunks reach the device on sp.copy and are decoded on sp.work.  Declare it inside the
// DevBufStreamScope of sp.work.
struct DeviceStaging {
  ChunkReader& rd;
  StreamPair& sp;
  std::vector<DevBuf<uint8_t>> dbuf;  // [ring]: LOAD_TILE bytes of slack, as the text kernels read whole tiles
  std::vector<cudaEvent_t> parsed;    // [ring]
  uint64_t h2d = 0;                   // bytes copied to the device

  DeviceStaging(ChunkReader& r, StreamPair& s) : rd(r), sp(s), dbuf(r.ring), parsed(r.ring, nullptr) {}
  gb_status create_events() {
    for (cudaEvent_t& e : parsed) GB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    return GB_OK;
  }
  ~DeviceStaging() {
    cudaStreamSynchronize(sp.copy);  // nothing may still be copying into dbuf when it is freed
    for (cudaEvent_t e : parsed)
      if (e) cudaEventDestroy(e);
  }

  // Copies cl carried bytes and then the first `body` bytes of chunk k (cl + body > 0) to the slot's staging
  // buffer, once the kernels that read it are done.  A carry that fits the LOAD_CARRY_RESERVE gap in front of
  // the pinned chunk goes with it in one copy; a longer one (a text line longer than the reserve) goes from
  // pageable memory.
  gb_status stage(uint64_t k, const char* carry, uint64_t cl, uint64_t body) {
    const unsigned r = (unsigned)(k % rd.ring);
    char* data = rd.data(r);
    const uint64_t len = cl + body;
    if (dbuf[r].n < len + LOAD_TILE) {
      GB_CUDA(cudaEventSynchronize(parsed[r]));
      DevBuf<uint8_t> nb;
      GB_TRY(nb.alloc(std::max<uint64_t>(len, rd.chunk + LOAD_CARRY_RESERVE) + LOAD_TILE));
      dbuf[r] = std::move(nb);
    }
    GB_CUDA(cudaStreamWaitEvent(sp.copy, parsed[r], 0));
    if (cl <= LOAD_CARRY_RESERVE) {
      std::memcpy(data - cl, carry, cl);
      GB_CUDA(cudaMemcpyAsync(dbuf[r].p, data - cl, len, cudaMemcpyHostToDevice, sp.copy));
    } else {
      GB_CUDA(cudaMemcpyAsync(dbuf[r].p, carry, cl, cudaMemcpyHostToDevice, sp.copy));
      if (body) GB_CUDA(cudaMemcpyAsync(dbuf[r].p + cl, data, body, cudaMemcpyHostToDevice, sp.copy));
    }
    h2d += len;
    return GB_OK;
  }
};

// grows a device array to hold at least `need` entries, keeping the first `keep`
template <typename T>
static gb_status grow(DevBuf<T>& b, uint64_t need, uint64_t want, uint64_t keep, cudaStream_t s) {
  if (b.p && b.n >= need) return GB_OK;
  DevBuf<T> nb;
  GB_TRY(nb.alloc(std::max(need, want)));
  if (keep) GB_CUDA(cudaMemcpyAsync(nb.p, b.p, keep * sizeof(T), cudaMemcpyDeviceToDevice, s));
  b = std::move(nb);  // the old array is released once s has finished with it (DevBufStreamScope)
  return GB_OK;
}

struct LoadedEdges {
  DevBuf<uint32_t> src, dst;
  DevBuf<float> w;
  uint64_t m = 0;
  uint32_t n = 0;  // 0: max id + 1
};

static gb_status load_file(int device, const InputFile& f, gb_file_format format, bool want_value,
                           LoadedEdges* out, gb_load_info* info) {
  const bool g500 = format == GB_FORMAT_GRAPH500;
  ChunkReader rd(f.fd, device);
  const uint64_t m500 = f.bytes / 12;
  rd.plan(g500 ? 12 * m500 : f.bytes, g500 ? 48 : 1);  // Graph500: whole 4-record groups, a partial tail ignored
  info->chunks = rd.nchunks;
  if (rd.nchunks == 0) return GB_OK;  // empty: gb_*_from_device_edges reports it

  StreamPair sp;
  GB_CUDA(cudaStreamCreateWithFlags(&sp.copy, cudaStreamNonBlocking));
  GB_CUDA(cudaStreamCreateWithFlags(&sp.work, cudaStreamNonBlocking));
  GB_TRY(rd.start());
  DevBufStreamScope scope(sp.work);
  DeviceStaging st(rd, sp);
  GB_TRY(st.create_events());

  const unsigned R = rd.ring;
  DevBuf<LoadCounters> ctr;
  GB_TRY(ctr.alloc(1));
  GB_CUDA(cudaMemsetAsync(ctr.p, 0, sizeof(LoadCounters), sp.work));
  PinnedBuf small;  // [0] = '\n' in the chunk, [1] = declined so far
  GB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&small.p), 64, cudaHostAllocDefault));
  uint32_t* hsmall = reinterpret_cast<uint32_t*>(small.p);

  DevBuf<uint32_t> counts;  // per-tile '\n' counts, scanned in place
  DevBuf<uint8_t> scan_tmp;
  DevBuf<uint64_t> dec_off;
  DevBuf<uint32_t> dec_edge;
  uint64_t m = 0;
  if (g500) {
    GB_TRY(out->src.alloc(m500));
    GB_TRY(out->dst.alloc(m500));
  }

  // what prepare() leaves for run(): the device chunk and where it starts in the file
  struct Staged {
    uint64_t len = 0, file_off = 0;
    bool ends_with_newline = true;
  };
  std::vector<Staged> staged(R);
  std::string carry;  // text: the bytes after the last '\n' so far

  // waits for chunk k's bytes, moves them (with the carried line in front) to the device on the copy stream
  auto prepare = [&](uint64_t k) -> gb_status {
    const unsigned r = (unsigned)(k % R);
    GB_TRY(rd.wait_filled(k));
    const char* data = rd.data(r);
    const uint64_t n = rd.chunk_bytes(k);
    const bool last = k + 1 == rd.nchunks;
    uint64_t body = n;  // bytes of this chunk that go to the device now
    std::string next_carry;
    if (!g500 && !last) {
      const void* nl = memrchr(data, '\n', n);
      body = nl ? (uint64_t)(static_cast<const char*>(nl) - data) + 1 : 0;
      if (!nl) next_carry = carry;
      next_carry.append(data + body, n - body);
    }
    const uint64_t cl = (!g500 && (body || last)) ? carry.size() : 0;  // carried bytes that go in front
    Staged& sg = staged[r];
    sg.len = cl + body;
    sg.file_off = k * rd.chunk - cl;
    sg.ends_with_newline = sg.len == 0 || (body ? data[body - 1] == '\n' : carry.back() == '\n');
    if (sg.len) GB_TRY(st.stage(k, carry.data(), cl, body));
    GB_TRY(rd.release(k, sp));
    if (!g500) carry.swap(next_carry);
    return GB_OK;
  };

  GB_TRY(prepare(0));
  for (uint64_t k = 0; k < rd.nchunks; ++k) {
    const unsigned r = (unsigned)(k % R);
    const Staged sg = staged[r];
    const uint4* d = reinterpret_cast<const uint4*>(st.dbuf[r].p);
    if (g500) {
      if (k + 1 < rd.nchunks) GB_TRY(prepare(k + 1));
      const uint64_t nrec = sg.len / 12;
      if (nrec) {
        k_load_graph500<<<grid_for((nrec + 3) / 4, 256), 256, 0, sp.work>>>(d, nrec, k * rd.chunk / 12, out->src.p,
                                                                             out->dst.p, ctr.p);
        GB_CUDA(cudaGetLastError());
      }
      GB_CUDA(cudaEventRecord(st.parsed[r], sp.work));
      continue;
    }
    const uint64_t tiles = (sg.len + LOAD_TILE - 1) / LOAD_TILE;
    if (tiles) {
      GB_TRY(grow(counts, tiles, 2 * tiles, 0, sp.work));
      k_load_count_lines<<<(unsigned)tiles, LOAD_BLOCK, 0, sp.work>>>(d, sg.len, counts.p);
      GB_TRY(cub_call(scan_tmp, [&](void* t, size_t& tb) {
        return cub::DeviceScan::InclusiveSum(t, tb, counts.p, counts.p, (int)tiles, sp.work);
      }, 2));
      GB_CUDA(cudaMemcpyAsync(hsmall, counts.p + tiles - 1, 4, cudaMemcpyDeviceToHost, sp.work));
      GB_CUDA(cudaMemcpyAsync(hsmall + 1, &ctr.p->declined, 4, cudaMemcpyDeviceToHost, sp.work));
    }
    if (k + 1 < rd.nchunks) GB_TRY(prepare(k + 1));  // the next chunk crosses the bus meanwhile
    if (tiles) {
      GB_CUDA(cudaStreamSynchronize(sp.work));
      const uint64_t lines = hsmall[0] + (sg.ends_with_newline ? 0 : 1);
      // size the arrays for the whole file from the lines per byte seen so far
      const uint64_t through = std::min(rd.read_end, (k + 1) * rd.chunk);
      const uint64_t est = (uint64_t)((double)(m + lines) * (double)rd.read_end / (double)through * 1.02) + 1024;
      const uint64_t want = std::max(est, out->src.n + out->src.n / 2);
      GB_TRY(grow(out->src, m + lines, want, m, sp.work));
      GB_TRY(grow(out->dst, m + lines, want, m, sp.work));
      if (want_value) {
        GB_TRY(grow(out->w, m + lines, want, m, sp.work));
        const uint64_t declined = hsmall[1];
        GB_TRY(grow(dec_off, declined + lines, 2 * (declined + lines), declined, sp.work));
        GB_TRY(grow(dec_edge, declined + lines, 2 * (declined + lines), declined, sp.work));
      }
      k_load_parse_text<<<(unsigned)tiles, LOAD_BLOCK, 0, sp.work>>>(d, sg.len, counts.p, m, sg.file_off,
                                                                    want_value ? 1 : 0, out->src.p, out->dst.p,
                                                                    out->w.p, ctr.p, dec_off.p, dec_edge.p);
      GB_CUDA(cudaGetLastError());
      m += lines;
    }
    GB_CUDA(cudaEventRecord(st.parsed[r], sp.work));
  }
  LoadCounters hc{};
  GB_CUDA(cudaMemcpyAsync(&hc, ctr.p, sizeof hc, cudaMemcpyDeviceToHost, sp.work));
  GB_CUDA(cudaStreamSynchronize(sp.work));
  GB_REQUIRE(hc.wide == 0, g500 ? "Graph500 node id does not fit 32 bits" : "edge list node id does not fit 32 bits");
  if (g500) m = m500;

  // declined values: re-read each line and parse it with the host reader's own function
  if (hc.declined) {
    std::vector<uint64_t> off(hc.declined);
    std::vector<uint32_t> edge(hc.declined);
    GB_CUDA(cudaMemcpyAsync(off.data(), dec_off.p, hc.declined * 8ull, cudaMemcpyDeviceToHost, sp.work));
    GB_CUDA(cudaMemcpyAsync(edge.data(), dec_edge.p, hc.declined * 4ull, cudaMemcpyDeviceToHost, sp.work));
    GB_CUDA(cudaStreamSynchronize(sp.work));
    std::vector<float> val(hc.declined);
    std::string line;
    for (uint64_t i = 0; i < hc.declined; ++i) {
      uint64_t want = 256;
      for (;;) {
        const uint64_t n = std::min(want, f.bytes - off[i]);
        line.resize(n);
        if (!pread_all(f.fd, &line[0], n, off[i])) return fail(GB_ERR_INVALID, "reading %s failed", f.path);
        if (n == f.bytes - off[i] || std::memchr(line.data(), '\n', n)) break;
        want *= 2;
      }
      uint64_t s, t;
      gb::parse_line(line.data(), 0, line.size(), 1, &s, &t, &val[i]);
    }
    DevBuf<float> dval;
    GB_TRY(dval.alloc(hc.declined));
    GB_CUDA(cudaMemcpyAsync(dval.p, val.data(), hc.declined * 4ull, cudaMemcpyHostToDevice, sp.work));
    k_load_patch<<<grid_for(hc.declined, 256), 256, 0, sp.work>>>(dec_edge.p, dval.p, hc.declined, out->w.p);
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaStreamSynchronize(sp.work));
    st.h2d += hc.declined * 4ull;
  }
  out->m = m;
  out->n = g500 ? (uint32_t)std::min<uint64_t>(m500 / 16, 0xFFFFFFFFull) : 0;  // graph500.rs:74
  info->edges = m;
  info->fallback_lines = hc.declined;
  info->h2d_bytes = st.h2d;
  GB_CUDA(cudaStreamSynchronize(sp.copy));
  return GB_OK;
}

// The CSR arrays a binary file's section fills.  Elements of `stride` bytes start at file byte `pos`; a u32
// section without values (stride 4) is DMA'd straight into `ids`, the others are staged and split by
// k_bin_split.
struct BinSection {
  uint64_t pos = 0, count = 0;
  uint32_t stride = 0;
  uint32_t* ids = nullptr;
  float* w = nullptr;
  bool direct() const { return stride == 4; }
  uint64_t end() const { return pos + count * stride; }
};

// the checks of gb_binary_decode on the device arrays: offsets[0] == 0, monotone, offsets[n] == entries, targets
// below n; `wide` is the flag of the narrowing kernel
static gb_status check_loaded_csrs(gb_graph* g, const BinLayout& l, DevCsr* const* csr, unsigned int* d_wide,
                                   cudaStream_t s) {
  DevBuf<unsigned int> bad;  // per CSR: [2c] targets >= n, [2c + 1] decreasing rows
  DevBuf<uint32_t> ends;     // per CSR: offsets[0], offsets[n]
  GB_TRY(bad.alloc(4));
  GB_TRY(ends.alloc(4));
  GB_CUDA(cudaMemsetAsync(bad.p, 0, 16, s));
  for (unsigned c = 0; c < l.ncsr; ++c) {
    check_ids_async(s, csr[c]->tgt.p, l.entries, l.n, bad.p + 2 * c);
    check_monotone_async(s, csr[c]->off.p, l.n, bad.p + 2 * c + 1);
    GB_CUDA(cudaMemcpyAsync(ends.p + 2 * c, csr[c]->off.p, 4, cudaMemcpyDeviceToDevice, s));
    GB_CUDA(cudaMemcpyAsync(ends.p + 2 * c + 1, csr[c]->off.p + l.n, 4, cudaMemcpyDeviceToDevice, s));
  }
  GB_CUDA(cudaGetLastError());
  unsigned int h[5] = {0, 0, 0, 0, 0};
  uint32_t e[4] = {0, 0, 0, 0};
  GB_CUDA(cudaMemcpyAsync(h, bad.p, 16, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaMemcpyAsync(h + 4, d_wide, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaMemcpyAsync(e, ends.p, 16, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  GB_REQUIRE(h[4] == 0, "binary graph file: an id or offset does not fit 32 bits");
  for (unsigned c = 0; c < l.ncsr; ++c) {
    const char* what = bin_csr_name(l, c);
    GB_REQUIRE(e[2 * c] == 0, "%s offsets[0] must be 0", what);
    GB_TRY(require_monotone(what, h[2 * c + 1]));
    GB_REQUIRE(e[2 * c + 1] == l.entries, "%s offsets end at %u, not at its %llu entries", what, e[2 * c + 1],
               (unsigned long long)l.entries);
    GB_TRY(require_ids(what, h[2 * c], g->n));
  }
  return GB_OK;
}

// Binary graph files streamed into the CSR arrays.  A staged chunk carries at most 15 bytes of a cut element
// in front, and k_bin_split decodes the elements that end inside the chunk.
static gb_status load_binary_streamed(int device, gb_graph_kind kind, const InputFile& f, bool want_value,
                                      gb_graph** graph, gb_load_info* info) {
  BinLayout l;
  GB_TRY(bin_parse([&](uint64_t pos, void* dst, uint64_t n) { return pread_all(f.fd, static_cast<char*>(dst), n, pos); },
                   f.bytes, kind, &l));
  GB_REQUIRE(!want_value || l.values, "the binary graph file holds no edge values");
  GraphPtr g;
  GB_TRY(new_graph(device, kind, l.n, &g));

  StreamPair sp;
  GB_CUDA(cudaStreamCreateWithFlags(&sp.copy, cudaStreamNonBlocking));
  GB_CUDA(cudaStreamCreateWithFlags(&sp.work, cudaStreamNonBlocking));
  DevBufStreamScope scope(sp.work);
  DevCsr* csr[2] = {&g->out, &g->in};
  std::vector<BinSection> secs;
  for (unsigned c = 0; c < l.ncsr; ++c) {
    DevCsr& d = *csr[c];
    d.len = l.entries;
    GB_TRY(d.off.alloc((size_t)l.n + 1));
    GB_TRY(d.tgt.alloc(l.entries, 8));
    GB_CUDA(cudaMemsetAsync(d.tgt.p + l.entries, 0, 8 * 4, sp.work));
    if (c == 0 && want_value) GB_TRY(d.w.alloc(l.entries, 8));  // only a digraph's out-CSR keeps values
    BinSection o, t;
    o.pos = l.csr[c].off_pos, o.count = (uint64_t)l.n + 1, o.stride = l.id_bytes, o.ids = d.off.p;
    t.pos = l.csr[c].rec_pos, t.count = l.entries, t.stride = l.rec_bytes, t.ids = d.tgt.p, t.w = d.w.p;
    secs.push_back(o);
    if (t.count) secs.push_back(t);
  }

  ChunkReader rd(f.fd, device);
  rd.plan(f.bytes);
  info->chunks = rd.nchunks;
  GB_TRY(rd.start());
  DeviceStaging st(rd, sp);
  GB_TRY(st.create_events());
  const unsigned R = rd.ring;
  DevBuf<unsigned int> wide;
  GB_TRY(wide.alloc(1));
  GB_CUDA(cudaMemsetAsync(wide.p, 0, 4, sp.work));

  std::vector<uint64_t> staged_off(R, 0);  // file byte of st.dbuf[r][0], or ~0: the chunk was not staged
  std::string carry;                       // bytes of the staged element that the next chunk completes
  auto prepare = [&](uint64_t k) -> gb_status {
    const unsigned r = (unsigned)(k % R);
    GB_TRY(rd.wait_filled(k));
    const char* data = rd.data(r);
    const uint64_t a = k * rd.chunk, len = rd.chunk_bytes(k), b = a + len;
    bool stage = false;
    for (const BinSection& s : secs) stage |= !s.direct() && s.pos < b && s.end() > a;
    const uint64_t cl = stage ? carry.size() : 0;
    staged_off[r] = stage ? a - cl : ~0ull;
    if (stage) GB_TRY(st.stage(k, carry.data(), cl, len));
    for (const BinSection& s : secs) {
      if (!s.direct()) continue;
      const uint64_t x = std::max(a, s.pos), y = std::min(b, s.end());
      if (x >= y) continue;
      GB_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(s.ids) + (x - s.pos), data + (x - a), y - x,
                              cudaMemcpyHostToDevice, sp.copy));
      st.h2d += y - x;
    }
    carry.clear();
    for (const BinSection& s : secs)
      if (!s.direct() && s.pos < b && s.end() > b) {
        const uint64_t cut = (b - s.pos) % s.stride;  // bytes of the element that begins before b
        carry.assign(data + (len - cut), cut);
      }
    return rd.release(k, sp);
  };
  auto split = [&](uint64_t k) -> gb_status {
    const unsigned r = (unsigned)(k % R);
    if (staged_off[r] == ~0ull) return GB_OK;
    const uint64_t a = k * rd.chunk, b = a + rd.chunk_bytes(k);
    for (const BinSection& s : secs) {
      if (s.direct() || s.pos >= b || s.end() <= a) continue;
      const uint64_t first = a > s.pos ? (a - s.pos) / s.stride : 0;  // the first element that ends after a
      const uint64_t last = std::min(s.count, (b - s.pos) / s.stride);  // elements that end by b
      if (last <= first) continue;
      k_bin_split<<<grid_for(last - first, 256), 256, 0, sp.work>>>(st.dbuf[r].p, staged_off[r], s.pos, s.stride,
                                                                      l.id_bytes, first, last - first, s.ids, s.w,
                                                                      wide.p);
      GB_CUDA(cudaGetLastError());
    }
    GB_CUDA(cudaEventRecord(st.parsed[r], sp.work));
    return GB_OK;
  };
  GB_TRY(prepare(0));
  for (uint64_t k = 0; k < rd.nchunks; ++k) {
    if (k + 1 < rd.nchunks) GB_TRY(prepare(k + 1));  // the next chunk crosses the bus meanwhile
    GB_TRY(split(k));
  }
  GB_CUDA(cudaStreamSynchronize(sp.copy));
  GB_TRY(check_loaded_csrs(g.get(), l, csr, wide.p, sp.work));
  info->edges = kind == GB_KIND_DIRECTED ? l.entries : l.entries / 2;
  info->h2d_bytes = st.h2d;
  *graph = g.release();
  return GB_OK;
}

// Below these sizes the fixed costs of the pipeline (threads, streams, pinned ring) exceed what it saves, and
// the host readers are faster (H100 80GB HBM3, 400 W; tools/bench_load.py).  GB_LOAD_CHUNK_BYTES, when
// set, selects the device path whatever the size.
constexpr uint64_t LOAD_DEVICE_MIN_BYTES = 64ull << 20;

// the host readers of io.cu and the upload of gb_[di]graph_from_edges_u32
static gb_status load_on_host(int device, gb_graph_kind kind, const InputFile& f, gb_file_format format,
                              gb_layout layout, bool want_value, gb_graph** graph, gb_load_info* info) {
  std::unique_ptr<char[]> bytes;
  GB_TRY(f.read_all(&bytes));
  const uint64_t len = f.bytes;
  std::vector<uint32_t> src, dst;
  std::vector<float> w;
  uint64_t m = 0;
  uint32_t n = 0;
  if (format == GB_FORMAT_GRAPH500) {
    src.resize(len / 12);
    dst.resize(len / 12);
    GB_TRY(gb_graph500_decode(bytes.get(), len, src.data(), dst.data(), &m, &n));
  } else {
    GB_TRY(gb_edge_list_parse(bytes.get(), len, nullptr, nullptr, nullptr, &m));
    src.resize(m);
    dst.resize(m);
    if (want_value) w.resize(m);
    GB_TRY(gb_edge_list_parse(bytes.get(), len, src.data(), dst.data(), want_value ? w.data() : nullptr, &m));
  }
  if (kind == GB_KIND_DIRECTED)
    GB_TRY(gb_digraph_from_edges_u32(device, src.data(), dst.data(), want_value ? w.data() : nullptr, m, n, layout,
                                     graph));
  else
    GB_TRY(gb_graph_from_edges_u32(device, src.data(), dst.data(), m, n, layout, graph));
  info->edges = m;
  info->h2d_bytes = m * (want_value ? 12 : 8);
  return GB_OK;
}

// a small binary file: gb_binary_decode, then the upload of gb_[di]graph_from_csr_u32
static gb_status load_binary_on_host(int device, gb_graph_kind kind, const InputFile& f, bool want_value,
                                     gb_graph** graph, gb_load_info* info) {
  std::unique_ptr<char[]> bytes;
  GB_TRY(f.read_all(&bytes));
  const uint64_t len = f.bytes;
  uint32_t n = 0;
  uint64_t m = 0;
  int has_values = 0;
  GB_TRY(gb_binary_decode(bytes.get(), len, kind, &n, &m, &has_values, nullptr, nullptr, nullptr, nullptr, nullptr));
  GB_REQUIRE(!want_value || has_values, "the binary graph file holds no edge values");
  const unsigned ncsr = kind == GB_KIND_DIRECTED ? 2 : 1;
  std::vector<uint32_t> off[2], tgt[2];
  std::vector<float> w(want_value ? m : 0);
  for (unsigned c = 0; c < ncsr; ++c) off[c].resize((size_t)n + 1), tgt[c].resize(m);
  GB_TRY(gb_binary_decode(bytes.get(), len, kind, &n, &m, &has_values, off[0].data(), tgt[0].data(),
                          want_value ? w.data() : nullptr, off[1].data(), tgt[1].data()));
  GraphPtr g;
  GB_TRY(new_graph(device, kind, n, &g));
  GB_TRY(upload_host_csr(g->stream, n, off[0].data(), tgt[0].data(), want_value ? w.data() : nullptr, &g->out,
                         kind == GB_KIND_DIRECTED ? "csr_out" : "csr"));
  if (kind == GB_KIND_DIRECTED)
    GB_TRY(upload_host_csr(g->stream, n, off[1].data(), tgt[1].data(), nullptr, &g->in, "csr_inc"));
  *graph = g.release();
  info->edges = kind == GB_KIND_DIRECTED ? m : m / 2;
  info->h2d_bytes = ncsr * (((uint64_t)n + 1) * 4 + m * 4) + (want_value ? m * 4 : 0);
  return GB_OK;
}

static bool pwrite_all(int fd, const char* src, uint64_t bytes, uint64_t off) {
  while (bytes) {
    const ssize_t r = ::pwrite(fd, src, bytes, (off_t)off);
    if (r < 0 && errno == EINTR) continue;
    if (r <= 0) return false;
    src += r;
    off += (uint64_t)r;
    bytes -= (uint64_t)r;
  }
  return true;
}

// the file being written; removed unless it was renamed over the destination
struct TempFile {
  std::string path;
  int fd = -1;
  bool renamed = false;
  ~TempFile() {
    if (fd >= 0) ::close(fd);
    if (!renamed && !path.empty()) ::unlink(path.c_str());
  }
};

// SerializeGraphOp::serialize (headers from host memory, arrays from device memory; Target<u32, f32> records are
// interleaved on the device first)
static gb_status serialize_graph(const gb_graph* g, const char* path) {
  GB_REQUIRE(g && path, "NULL argument");
  GB_REQUIRE(g->out.tgt.p != nullptr, "this handle holds no out targets (page-rank-only twin) and cannot be serialized");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  const bool values = g->kind == GB_KIND_DIRECTED && g->out.w.p != nullptr;
  const BinLayout l = bin_layout_u32(g->kind, g->n, g->out.len, values);
  const DevCsr* csr[2] = {&g->out, &g->in};
  DevBuf<float> in_w;
  if (values) GB_TRY(in_csr_values(g, &in_w));
  struct Piece {
    uint64_t pos, len;
    const void* src;
    bool device;
  };
  std::vector<Piece> pieces;
  std::string headers[2];
  DevBuf<uint2> records[2];
  for (unsigned c = 0; c < l.ncsr; ++c) {
    headers[c] = bin_header_bytes(l, c);
    pieces.push_back({c == 0 ? 0 : l.csr[c].header, headers[c].size(), headers[c].data(), false});
    pieces.push_back({l.csr[c].off_pos, ((uint64_t)l.n + 1) * 4, csr[c]->off.p, true});
    if (!l.entries) continue;
    if (values) {
      GB_TRY(records[c].alloc(l.entries));
      k_bin_interleave<<<grid_for(l.entries, 256), 256, 0, g->stream>>>(csr[c]->tgt.p, c == 0 ? g->out.w.p : in_w.p,
                                                                         l.entries, records[c].p);
      GB_CUDA(cudaGetLastError());
      pieces.push_back({l.csr[c].rec_pos, l.entries * 8, records[c].p, true});
    } else {
      pieces.push_back({l.csr[c].rec_pos, l.entries * 4, csr[c]->tgt.p, true});
    }
  }
  GB_CUDA(cudaStreamSynchronize(g->stream));

  TempFile tmp;
  tmp.path = std::string(path) + ".XXXXXX";
  tmp.fd = ::mkstemp(&tmp.path[0]);
  if (tmp.fd < 0) {
    tmp.path.clear();
    return fail(GB_ERR_INVALID, "cannot create a temporary file next to %s: %s", path, std::strerror(errno));
  }
  ::fchmod(tmp.fd, 0644);
  PinnedRing ring;
  ring.plan(l.file_bytes);  // ring >= 2 whenever there is a next chunk
  GB_TRY(ring.acquire());
  StreamPair sp;
  GB_CUDA(cudaStreamCreateWithFlags(&sp.copy, cudaStreamNonBlocking));
  auto fill = [&](uint64_t k) -> gb_status {
    const unsigned r = (unsigned)(k % ring.ring);
    char* data = ring.data(r);
    const uint64_t a = k * ring.chunk, b = a + ring.chunk_bytes(k);
    for (const Piece& p : pieces) {
      const uint64_t x = std::max(a, p.pos), y = std::min(b, p.pos + p.len);
      if (x >= y) continue;
      const char* src = static_cast<const char*>(p.src) + (x - p.pos);
      if (p.device) GB_CUDA(cudaMemcpyAsync(data + (x - a), src, y - x, cudaMemcpyDeviceToHost, sp.copy));
      else std::memcpy(data + (x - a), src, y - x);
    }
    GB_CUDA(cudaEventRecord(ring.copied[r], sp.copy));
    return GB_OK;
  };
  GB_TRY(fill(0));
  for (uint64_t k = 0; k < ring.nchunks; ++k) {
    if (k + 1 < ring.nchunks) GB_TRY(fill(k + 1));  // its buffer was written out R - 1 chunks ago
    const unsigned r = (unsigned)(k % ring.ring);
    GB_CUDA(cudaEventSynchronize(ring.copied[r]));
    if (!pwrite_all(tmp.fd, ring.data(r), ring.chunk_bytes(k), k * ring.chunk))
      return fail(GB_ERR_INVALID, "writing %s failed: %s", tmp.path.c_str(), std::strerror(errno));
  }
  const int fd = tmp.fd;
  tmp.fd = -1;
  if (::close(fd) != 0) return fail(GB_ERR_INVALID, "writing %s failed: %s", tmp.path.c_str(), std::strerror(errno));
  if (::rename(tmp.path.c_str(), path) != 0)
    return fail(GB_ERR_INVALID, "cannot rename %s to %s: %s", tmp.path.c_str(), path, std::strerror(errno));
  tmp.renamed = true;
  return GB_OK;
}

static gb_status load_graph(int device, gb_graph_kind kind, const char* path, gb_file_format format,
                            gb_layout layout, int with_values, gb_graph** graph) {
  GB_REQUIRE(graph != nullptr, "graph out-pointer is NULL");
  GB_REQUIRE(path != nullptr, "path is NULL");
  GB_REQUIRE(format == GB_FORMAT_GRAPH500 || format == GB_FORMAT_EDGE_LIST || format == GB_FORMAT_BINARY,
             "unknown file format %d", (int)format);
  GB_REQUIRE(!with_values || format != GB_FORMAT_GRAPH500, "only edge lists and binary files carry edge values");
  GB_TRY(check_layout(layout));
  GB_TRY(require_device(device));
  DeviceGuard guard(device);
  InputFile f;
  GB_TRY(f.open(path));
  gb_load_info info{};
  info.file_bytes = f.bytes;
  const bool on_host = env_chunk_bytes() == 0 && f.bytes < LOAD_DEVICE_MIN_BYTES;
  if (format == GB_FORMAT_BINARY) {
    if (on_host) GB_TRY(load_binary_on_host(device, kind, f, with_values != 0, graph, &info));
    else GB_TRY(load_binary_streamed(device, kind, f, with_values != 0, graph, &info));
  } else if (on_host) {
    GB_TRY(load_on_host(device, kind, f, format, layout, with_values != 0, graph, &info));
  } else {
    LoadedEdges e;
    GB_TRY(load_file(device, f, format, with_values != 0, &e, &info));
    GB_TRY(graph_from_device_arrays(device, kind, e.src.p, e.dst.p, with_values ? e.w.p : nullptr, e.m, e.n, layout,
                                    nullptr, graph));
  }
  (*graph)->load = info;
  return GB_OK;
}

}  // namespace gb

extern "C" {

gb_status gb_digraph_load_u32(int device, const char* path, gb_file_format format, gb_layout layout,
                              int with_values, gb_graph** graph) {
  return gb::load_graph(device, GB_KIND_DIRECTED, path, format, layout, with_values, graph);
}

gb_status gb_graph_load_u32(int device, const char* path, gb_file_format format, gb_layout layout,
                            gb_graph** graph) {
  return gb::load_graph(device, GB_KIND_UNDIRECTED, path, format, layout, 0, graph);
}

gb_status gb_graph_serialize(const gb_graph* graph, const char* path) { return gb::serialize_graph(graph, path); }

gb_status gb_graph_load_info(const gb_graph* g, gb_load_info* info) {
  GB_REQUIRE(g && info, "NULL argument");
  *info = g->load;
  return GB_OK;
}

}  // extern "C"
