// load.cu — graph files streamed between the file and device memory: Graph500 and text edge lists parsed into
// device edge arrays, and binary CSR files read into and written from the device CSR arrays.
//
// load_graph opens the file once.  Below LOAD_DEVICE_MIN_BYTES the host decoders of io.cu read it whole in
// pageable memory and their result is uploaded.  Larger files go through a ring of pinned buffers
// (PinnedRing): chunk k of the file travels through buffer k % ring.  On a load, one reader thread per buffer
// preads the chunks that map to it (ChunkReader), a copy stream moves each chunk to the device slot's staging
// buffer (DeviceStaging), and kernels on a work stream decode it; stream_file runs that loop, and one decoder per
// format below says what each chunk stages and decodes.  On a save the copy stream fills the buffers from device
// memory and the host writes them out.  Ordering rules:
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
//   DotGraph: the text pipeline above, with the line index of every line.  The host reads the header "t N M" first;
//   k_load_parse_dotgraph sends line 1..N to labels[line - 1] and line N+1..N+M to src / dst[line - 1 - N]
//   (dotgraph_line.h), ignores the lines after them, and keeps the smallest (line, error) pair it meets.
//   Binary: the host preads the headers (bin_parse gives the section table) and every chunk is cut against the
//   table.  u32 sections without values go from the pinned buffer straight into their CSR array; a chunk that
//   meets another section is staged with the bytes of the element it cuts carried in front, and k_bin_split
//   narrows the ids and splits the records.  A labelled file's NodeValues are one more section: 4-byte labels go
//   straight into the label array, 8-byte ones are narrowed by k_bin_split, which keeps the smallest node whose
//   label does not fit 32 bits.
//   Writer: the file is pieces of host and device memory; chunk k + 1 is copied from the device into the ring
//   while chunk k is written with pwrite to a temporary file, which is then renamed over the destination.
//   WCC of a file (gb_wcc_file_u32): the same decoders, given a WccSink, decode each chunk into per-chunk scratch
//   instead of whole-file arrays and hand it to the sink, which links it into a parent array (DESIGN.md §11).
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

// the labels of a gb_wcc_file_u32 call, on the device that computed them
struct gb_components {
  int device = 0;
  uint32_t n = 0;
  gb::DevBuf<uint32_t> labels;
};

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

// DotGraph lines (dotgraph_line.h), found as k_load_parse_text finds them; line_base = lines of the earlier chunks,
// with the header as line 0.  The first error (smallest line) is kept as line << 3 | code in *first_error.  A NULL
// labels (or src, and with it dst) skips those stores.
__global__ void __launch_bounds__(LOAD_BLOCK) k_load_parse_dotgraph(const uint4* __restrict__ buf, uint64_t len,
                                                                    const uint32_t* __restrict__ incl,
                                                                    uint64_t line_base, uint32_t nodes,
                                                                    uint64_t lines, uint32_t* __restrict__ labels,
                                                                    uint32_t* __restrict__ src,
                                                                    uint32_t* __restrict__ dst,
                                                                    unsigned long long* __restrict__ first_error) {
  using Scan = cub::BlockScan<uint32_t, LOAD_BLOCK>;
  __shared__ typename Scan::TempStorage tmp;
  const uint64_t i = (uint64_t)blockIdx.x * LOAD_BLOCK + threadIdx.x;
  const uint64_t pos = 16 * i;
  uint32_t m = newline_mask(buf[i], pos, len);
  uint32_t before;
  Scan(tmp).ExclusiveSum((uint32_t)__popc(m), before);
  uint64_t line = line_base + (blockIdx.x ? incl[blockIdx.x - 1] : 0u) + before;
  const char* text = reinterpret_cast<const char*>(buf);
  auto parse = [&](uint64_t start, uint64_t ln) {
    if (ln == 0 || ln >= lines) return;
    uint64_t eol = start;
    while (eol < len && text[eol] != '\n') ++eol;
    uint32_t v[3];
    const bool node = ln <= nodes;
    const uint32_t code = dot_line(text, start, eol, node ? 3 : 2, v);
    if (code) {
      atomicMin(first_error, (unsigned long long)(ln << 3 | code));
    } else if (node) {
      if (labels) labels[ln - 1] = v[1];
    } else if (src) {
      src[ln - 1 - nodes] = v[0];
      dst[ln - 1 - nodes] = v[1];
    }
  };
  if (i == 0 && len > 0) parse(0, line_base);
  while (m) {
    const int j = __ffs(m) - 1;
    m &= m - 1;
    ++line;
    if (pos + j + 1 < len) parse(pos + j + 1, line);
  }
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
// that is not 0 sets *wide), followed by an f32 value that goes to w[e] when w is not NULL.  With first_wide
// (the labels, whose elements number below 2^32) the smallest such e goes to *first_wide instead of the flag.
__global__ void k_bin_split(const uint8_t* __restrict__ buf, uint64_t buf_off, uint64_t sec, uint32_t stride,
                            uint32_t id_bytes, uint64_t first, uint64_t count, uint32_t* __restrict__ ids,
                            float* __restrict__ w, unsigned int* __restrict__ wide,
                            unsigned int* __restrict__ first_wide) {
  bool big = false;
  unsigned int lo = 0xFFFFFFFFu;  // the first e of this thread with a high word (its e ascend)
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t e = first + i;
    const uint64_t pos = sec + e * stride - buf_off;
    ids[e] = load_u32_at(buf, pos);
    if (id_bytes == 8 && load_u32_at(buf, pos + 4) != 0) {
      if (!big) lo = (unsigned int)e;
      big = true;
    }
    if (w) w[e] = __uint_as_float(load_u32_at(buf, pos + id_bytes));
  }
  if (first_wide) {
    lo = __reduce_min_sync(0xFFFFFFFFu, lo);
    if (lo != 0xFFFFFFFFu && (threadIdx.x & 31) == 0) atomicMin(first_wide, lo);
  } else if (__any_sync(0xFFFFFFFFu, big) && (threadIdx.x & 31) == 0) {
    atomicOr(wide, 1u);
  }
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
  // the bytes from `off` on through the next '\n' (or to the end of the file), read in pieces that start at
  // `piece` bytes and double until one holds the '\n'
  gb_status read_line(uint64_t off, uint64_t piece, std::string* out) const {
    for (;; piece *= 2) {
      const uint64_t n = std::min(piece, bytes - off);
      out->resize(n);
      if (!pread_all(fd, &(*out)[0], n, off)) return fail(GB_ERR_INVALID, "reading %s failed", path);
      if (n == bytes - off || std::memchr(out->data(), '\n', n)) return GB_OK;
    }
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

// The device side of a streamed load: per ring slot a staging buffer, what it holds, and the event recorded behind
// the kernels that read it.  Chunks reach the device on sp.copy and are decoded on sp.work.  Declare it inside the
// DevBufStreamScope of sp.work.
struct DeviceStaging {
  ChunkReader& rd;
  StreamPair& sp;
  std::vector<DevBuf<uint8_t>> dbuf;  // [ring]: LOAD_TILE bytes of slack, as the text kernels read whole tiles
  std::vector<uint64_t> off, len;     // [ring]: dbuf[r] holds len bytes from file byte off (len 0: none staged)
  std::vector<cudaEvent_t> parsed;    // [ring]
  uint64_t h2d = 0;                   // bytes copied to the device

  DeviceStaging(ChunkReader& r, StreamPair& s)
      : rd(r), sp(s), dbuf(r.ring), off(r.ring, 0), len(r.ring, 0), parsed(r.ring, nullptr) {}
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
    const uint64_t n = cl + body;
    if (dbuf[r].n < n + LOAD_TILE) {
      GB_CUDA(cudaEventSynchronize(parsed[r]));
      DevBuf<uint8_t> nb;
      GB_TRY(nb.alloc(std::max<uint64_t>(n, rd.chunk + LOAD_CARRY_RESERVE) + LOAD_TILE));
      dbuf[r] = std::move(nb);
    }
    GB_CUDA(cudaStreamWaitEvent(sp.copy, parsed[r], 0));
    if (cl <= LOAD_CARRY_RESERVE) {
      std::memcpy(data - cl, carry, cl);
      GB_CUDA(cudaMemcpyAsync(dbuf[r].p, data - cl, n, cudaMemcpyHostToDevice, sp.copy));
    } else {
      GB_CUDA(cudaMemcpyAsync(dbuf[r].p, carry, cl, cudaMemcpyHostToDevice, sp.copy));
      if (body) GB_CUDA(cudaMemcpyAsync(dbuf[r].p + cl, data, body, cudaMemcpyHostToDevice, sp.copy));
    }
    off[r] = k * rd.chunk - cl;
    len[r] = n;
    h2d += n;
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

// Chunk k of a streamed read: file bytes [a, b).  In a decoder's stage() they are in pinned memory at `data`; in
// its before() and after(), `dev` holds the len bytes that stage() sent to the device, from file byte `off`.
struct Chunk {
  uint64_t k, a, b;
  bool last;
  const char* data;
  const uint8_t* dev;
  uint64_t off, len;
};

// The consumer of decoded chunks behind gb_wcc_file_u32.  A decoder given one puts each chunk's edges into its
// scratch instead of whole-file arrays (src / dst pairs, or a binary chunk's targets in src) and hands them over in
// after(); they are linked into parent[] on the work stream s, behind the decode.  One scratch serves every chunk:
// chunk k's links run on s before the decode of chunk k + 1 overwrites it.  With no node_count up front (edge lists,
// DotGraph, Graph500 files of fewer than 16 records) it is the largest id so far + 1: each chunk's largest id is
// read back before its links, and parent[] grows by doubling with an identity tail.
struct WccSink {
  cudaStream_t s = nullptr;
  bool infer = true;          // node_count = max id + 1
  uint64_t n = 0, cap = 0;    // nodes so far, parent entries (the identity past n)
  bool max_id = false;        // an id 2^32 - 1 was read: no node_count fits
  bool stop = false;          // the read fails anyway: no more links
  DevBuf<uint32_t> parent;
  DevBuf<uint32_t> src, dst;  // one chunk's pairs; src holds a binary chunk's targets
  DevBuf<unsigned int> bad;   // pairs: [0] endpoints >= n; binary: [c] targets >= n of CSR c
  DevBuf<uint32_t> mx;        // the chunk's largest src and dst
  DevBuf<uint8_t> tmp;
  uint32_t host[3] = {0, 0, 0};
  cudaEvent_t begin = nullptr, end = nullptr;
  double total_ms = 0.0;
  // binary files: the offsets of the out- and in-CSR, and their checks (check_loaded_csrs's), made before the first
  // link searches them
  DevCsr csr[2];
  bool checked[2] = {false, false};
  uint32_t off_first[2] = {0, 0}, off_last[2] = {0, 0};
  unsigned int off_bad[2] = {0, 0};

  ~WccSink() {
    if (begin) cudaEventDestroy(begin);
    if (end) cudaEventDestroy(end);
  }
  // fixed_n: the file's node_count, or 0 when it is the largest id + 1
  gb_status start(cudaStream_t stream, uint64_t fixed_n) {
    s = stream;
    GB_CUDA(cudaEventCreate(&begin));
    GB_CUDA(cudaEventCreate(&end));
    GB_TRY(bad.alloc(2));
    GB_CUDA(cudaMemsetAsync(bad.p, 0, 8, s));
    GB_TRY(mx.alloc(2));
    infer = fixed_n == 0;
    if (!infer) {
      GB_TRY(parent.alloc(fixed_n));
      cc_init_async(s, parent.p, 0, fixed_n);
      n = cap = fixed_n;
    }
    return GB_OK;
  }
  // in a decoder's stage(): the timed section starts with chunk 0's first copy
  gb_status staging(const Chunk& c, cudaStream_t copy) {
    if (c.k == 0) GB_CUDA(cudaEventRecord(begin, copy));
    return GB_OK;
  }
  // room for `count` pairs (count targets when !pairs), with 8 entries of slack; a power of two, so that the
  // size follows the chunk size and not the file
  gb_status scratch(uint64_t count, bool pairs = true) {
    uint64_t want = 1024;
    while (want < count + 8) want *= 2;
    if (src.n < count + 8) GB_TRY(src.alloc(want));
    if (pairs && dst.n < count + 8) GB_TRY(dst.alloc(want));
    return GB_OK;
  }
  // links the `count` pairs the decoder has put into src / dst; d_stop: the decoder's flag of an error that fails
  // the read, read back with the largest id
  gb_status link_pairs(uint64_t count, const unsigned int* d_stop) {
    if (stop || count == 0) return GB_OK;
    if (infer) {
      GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) { return cub::DeviceReduce::Max(t, tb, src.p, mx.p, count, s); }));
      GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
        return cub::DeviceReduce::Max(t, tb, dst.p, mx.p + 1, count, s);
      }));
      host[2] = 0;
      GB_CUDA(cudaMemcpyAsync(host, mx.p, 8, cudaMemcpyDeviceToHost, s));
      if (d_stop) GB_CUDA(cudaMemcpyAsync(host + 2, d_stop, 4, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      const uint32_t hi = std::max(host[0], host[1]);
      max_id = hi == 0xFFFFFFFFu;
      if (host[2] || max_id) {
        stop = true;
        return GB_OK;
      }
      if (hi + 1ull > cap) {
        const uint64_t want = std::min<uint64_t>(std::max<uint64_t>(hi + 1ull, 2 * cap), 0xFFFFFFFFull);
        GB_TRY(grow(parent, hi + 1ull, want, cap, s));
        cc_init_async(s, parent.p, cap, parent.n);
        cap = parent.n;
      }
      n = std::max<uint64_t>(n, hi + 1ull);
    }
    cc_link_pairs_async(s, src.p, dst.p, count, (uint32_t)n, parent.p, bad.p);
    GB_CUDA(cudaGetLastError());
    return GB_OK;
  }
  // after the decoder's own checks: those of gb_[di]graph_from_device_edges_u32 on m edges (check_edge_args but
  // for the u32 offset limit, then check_edge_ids), and the labels
  gb_status finish_pairs(uint64_t m) {
    GB_REQUIRE(!infer || m > 0, "cannot infer node_count from an empty edge list");
    if (infer) {
      GB_REQUIRE(!max_id, "node id 2^32-1 leaves no room for node_count");
    } else {
      GB_CUDA(cudaMemcpyAsync(host, bad.p, 4, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      GB_REQUIRE(host[0] == 0, "%u edge endpoints are >= node_count %u", host[0], (uint32_t)n);
    }
    return finish();
  }
  // CSR c's offsets (all on the device): off[0], off[n] and the decreasing rows
  gb_status check_offsets(unsigned c, uint32_t rows) {
    if (checked[c]) return GB_OK;
    GB_CUDA(cudaMemsetAsync(mx.p, 0, 4, s));
    check_monotone_async(s, csr[c].off.p, rows, reinterpret_cast<unsigned int*>(mx.p));
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaMemcpyAsync(&off_bad[c], mx.p, 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaMemcpyAsync(&off_first[c], csr[c].off.p, 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaMemcpyAsync(&off_last[c], csr[c].off.p + rows, 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    checked[c] = true;
    return GB_OK;
  }
  // the targets [e0, e0 + count) of CSR c, which the decoder has put into src; not linked when c's offsets fail
  // their checks (the read fails on them, and the row searches need them)
  gb_status link_targets(unsigned c, const BinLayout& l, uint64_t e0, uint64_t count) {
    GB_TRY(check_offsets(c, l.n));
    if (off_first[c] != 0 || off_bad[c] != 0 || off_last[c] != l.entries) return GB_OK;
    cc_link_csr_async(s, csr[c].off.p, l.n, src.p, (uint32_t)e0, (uint32_t)count, parent.p, bad.p + c);
    GB_CUDA(cudaGetLastError());
    return GB_OK;
  }
  // the final compress; the scratch goes, parent[] stays for the caller
  gb_status finish() {
    cc_compress_async(s, parent.p, (uint32_t)n);
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaEventRecord(end, s));
    GB_CUDA(cudaStreamSynchronize(s));
    float ms = 0.0f;
    GB_CUDA(cudaEventElapsedTime(&ms, begin, end));
    total_ms = ms;
    src.release(), dst.release(), bad.release(), mx.release(), tmp.release();
    csr[0] = DevCsr(), csr[1] = DevCsr();
    return GB_OK;
  }
};

// The streamed read of a file, for every format: its first `bytes` in chunks of whole `unit`s (PinnedRing::plan),
// chunk k + 1 staged on sp.copy while chunk k is decoded on sp.work.  The Decoder is built here from sp.work and
// `args` (its leading fields) and supplies:
//   begin()        its arrays and counters, before the first chunk;
//   stage(c, st)   from chunk k's pinned bytes: st.stage of the carried bytes and a body, and direct copies on
//                  sp.copy (counted in st.h2d);
//   before(c)      the work it issues on sp.work before chunk k + 1 is prepared;
//   after(c)       the work it issues after that.  A chunk that staged nothing has neither;
//   finish(info)   its checks and results, once every chunk is decoded and sp.copy has drained.
// Destruction runs in reverse order of declaration, and the order matters:
//   - the decoder goes first, inside the DevBufStreamScope, so its arrays, like every array grown and replaced
//     during the read, are released in stream order on sp.work;
//   - ~DeviceStaging drains sp.copy before the staging buffers are freed;
//   - ~ChunkReader joins the reader threads before ~PinnedRing hands the pinned buffers back to PinnedRingCache.
template <typename Decoder, typename... Args>
static gb_status stream_file(int device, const InputFile& f, uint64_t bytes, uint64_t unit, gb_load_info* info,
                             Args&&... args) {
  ChunkReader rd(f.fd, device);
  rd.plan(bytes, unit);
  info->chunks = rd.nchunks;
  if (rd.nchunks == 0) return GB_OK;  // empty: gb_*_from_device_edges reports it

  StreamPair sp;
  GB_CUDA(cudaStreamCreateWithFlags(&sp.copy, cudaStreamNonBlocking));
  GB_CUDA(cudaStreamCreateWithFlags(&sp.work, cudaStreamNonBlocking));
  GB_TRY(rd.start());
  DevBufStreamScope scope(sp.work);
  DeviceStaging st(rd, sp);
  GB_TRY(st.create_events());
  Decoder dec{sp.work, std::forward<Args>(args)...};
  GB_TRY(dec.begin());

  auto chunk = [&](uint64_t k) {
    const unsigned r = (unsigned)(k % rd.ring);
    const uint64_t a = k * rd.chunk;
    return Chunk{k, a, a + rd.chunk_bytes(k), k + 1 == rd.nchunks, rd.data(r), st.dbuf[r].p, st.off[r], st.len[r]};
  };
  // waits for chunk k's bytes and lets the decoder move them to the device on the copy stream
  auto prepare = [&](uint64_t k) -> gb_status {
    GB_TRY(rd.wait_filled(k));
    st.len[k % rd.ring] = 0;
    GB_TRY(dec.stage(chunk(k), st));
    return rd.release(k, sp);
  };
  GB_TRY(prepare(0));
  for (uint64_t k = 0; k < rd.nchunks; ++k) {
    const Chunk c = chunk(k);
    if (c.len) GB_TRY(dec.before(c));
    if (k + 1 < rd.nchunks) GB_TRY(prepare(k + 1));  // the next chunk crosses the bus meanwhile
    if (c.len) {
      GB_TRY(dec.after(c));
      GB_CUDA(cudaEventRecord(st.parsed[k % rd.ring], sp.work));
    }
  }
  GB_CUDA(cudaStreamSynchronize(sp.copy));
  info->h2d_bytes = st.h2d;
  return dec.finish(info);
}

// Graph500 files, into arrays of m edges allocated up front, or chunk by chunk into the pairs of a WccSink
struct Graph500Decoder {
  cudaStream_t s;
  uint64_t m;  // records: a partial one at the end of the file is ignored
  EdgeArrays* out;
  WccSink* wcc = nullptr;  // instead of out
  DevBuf<LoadCounters> ctr;

  static uint32_t nodes(uint64_t m) { return (uint32_t)std::min<uint64_t>(m / 16, 0xFFFFFFFFull); }  // graph500.rs:74
  gb_status begin() {
    GB_TRY(ctr.alloc(1));
    GB_CUDA(cudaMemsetAsync(ctr.p, 0, sizeof(LoadCounters), s));
    if (wcc) return wcc->start(s, nodes(m));
    GB_TRY(out->src.alloc(m));
    GB_TRY(out->dst.alloc(m));
    return GB_OK;
  }
  gb_status stage(const Chunk& c, DeviceStaging& st) {
    if (wcc) GB_TRY(wcc->staging(c, st.sp.copy));
    return st.stage(c.k, "", 0, c.b - c.a);
  }
  gb_status before(const Chunk&) { return GB_OK; }
  gb_status after(const Chunk& c) {
    const uint64_t nrec = c.len / 12;  // >= 1: the file's first 12 m bytes are read
    if (wcc) {
      GB_TRY(wcc->scratch(nrec));
      k_load_graph500<<<grid_for((nrec + 3) / 4, 256), 256, 0, s>>>(reinterpret_cast<const uint4*>(c.dev), nrec, 0,
                                                                     wcc->src.p, wcc->dst.p, ctr.p);
      GB_CUDA(cudaGetLastError());
      return wcc->link_pairs(nrec, &ctr.p->wide);
    }
    k_load_graph500<<<grid_for((nrec + 3) / 4, 256), 256, 0, s>>>(reinterpret_cast<const uint4*>(c.dev), nrec,
                                                                   c.a / 12, out->src.p, out->dst.p, ctr.p);
    GB_CUDA(cudaGetLastError());
    return GB_OK;
  }
  gb_status finish(gb_load_info* info) {
    LoadCounters hc{};
    GB_CUDA(cudaMemcpyAsync(&hc, ctr.p, sizeof hc, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    GB_REQUIRE(hc.wide == 0, "Graph500 node id does not fit 32 bits");
    info->edges = m;
    if (wcc) return wcc->finish_pairs(m);
    out->m = m;
    out->n = nodes(m);
    return GB_OK;
  }
};

// The line-tile stage of the text formats: a chunk staged up to its last '\n' (the last chunk whole) with the
// carried bytes in front, then the tile counts and their scan into the tile bases the parse kernels take.
struct LineTiles {
  std::string carry;        // the bytes after the last '\n' so far
  bool open_end = false;    // the file's last byte is not a '\n': its last line has none
  DevBuf<uint32_t> counts;  // per-tile '\n' counts, scanned in place
  DevBuf<uint8_t> scan_tmp;
  PinnedBuf small;  // [0] = '\n' in the chunk; [1] is the edge-list decoder's
  uint32_t* host = nullptr;

  static uint64_t tiles(const Chunk& c) { return (c.len + LOAD_TILE - 1) / LOAD_TILE; }
  gb_status begin() {
    GB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&small.p), 64, cudaHostAllocDefault));
    host = reinterpret_cast<uint32_t*>(small.p);
    return GB_OK;
  }
  gb_status stage(const Chunk& c, DeviceStaging& st) {
    const uint64_t n = c.b - c.a;
    uint64_t body = n;  // bytes of this chunk that go to the device now
    if (c.last) {
      open_end = c.data[n - 1] != '\n';
    } else {
      const void* nl = memrchr(c.data, '\n', n);
      body = nl ? (uint64_t)(static_cast<const char*>(nl) - c.data) + 1 : 0;
    }
    if (body) {
      GB_TRY(st.stage(c.k, carry.data(), carry.size(), body));
      carry.clear();
    }
    carry.append(c.data + body, n - body);
    return GB_OK;
  }
  // enqueues the tile counts of the staged chunk, their scan and the copy of its '\n' count to host[0]
  gb_status count(const Chunk& c, cudaStream_t s) {
    const uint64_t t = tiles(c);
    GB_TRY(grow(counts, t, 2 * t, 0, s));
    k_load_count_lines<<<(unsigned)t, LOAD_BLOCK, 0, s>>>(reinterpret_cast<const uint4*>(c.dev), c.len, counts.p);
    GB_TRY(cub_call(scan_tmp, [&](void* tmp, size_t& tb) {
      return cub::DeviceScan::InclusiveSum(tmp, tb, counts.p, counts.p, (int)t, s);
    }, 2));
    GB_CUDA(cudaMemcpyAsync(host, counts.p + t - 1, 4, cudaMemcpyDeviceToHost, s));
    return GB_OK;
  }
  // the lines of the staged chunk, once host[0] has arrived
  uint64_t lines(const Chunk& c) const { return host[0] + (c.last && open_end ? 1 : 0); }
};

// Text edge lists, into arrays that grow as the lines come; the values the device parser declines are re-read
// on the host and patched in by k_load_patch once every chunk is parsed.
struct EdgeListDecoder {
  cudaStream_t s;
  const InputFile& f;
  bool want_value;
  EdgeArrays* out;
  WccSink* wcc = nullptr;  // instead of out (without values)
  LineTiles text;
  DevBuf<LoadCounters> ctr;
  DevBuf<uint64_t> dec_off;
  DevBuf<uint32_t> dec_edge;
  uint64_t m = 0;  // edges so far

  gb_status begin() {
    GB_TRY(ctr.alloc(1));
    GB_CUDA(cudaMemsetAsync(ctr.p, 0, sizeof(LoadCounters), s));
    if (wcc) GB_TRY(wcc->start(s, 0));
    return text.begin();
  }
  gb_status stage(const Chunk& c, DeviceStaging& st) {
    if (wcc) GB_TRY(wcc->staging(c, st.sp.copy));
    return text.stage(c, st);
  }
  gb_status before(const Chunk& c) {
    GB_TRY(text.count(c, s));
    GB_CUDA(cudaMemcpyAsync(text.host + 1, &ctr.p->declined, 4, cudaMemcpyDeviceToHost, s));
    return GB_OK;
  }
  gb_status after(const Chunk& c) {
    GB_CUDA(cudaStreamSynchronize(s));
    const uint64_t lines = text.lines(c);
    if (wcc) {
      GB_TRY(wcc->scratch(lines));
      k_load_parse_text<<<(unsigned)LineTiles::tiles(c), LOAD_BLOCK, 0, s>>>(
          reinterpret_cast<const uint4*>(c.dev), c.len, text.counts.p, 0, c.off, 0, wcc->src.p, wcc->dst.p, nullptr,
          ctr.p, nullptr, nullptr);
      GB_CUDA(cudaGetLastError());
      m += lines;
      return wcc->link_pairs(lines, &ctr.p->wide);
    }
    // size the arrays for the whole file from the lines per byte seen so far
    const uint64_t est = (uint64_t)((double)(m + lines) * (double)f.bytes / (double)c.b * 1.02) + 1024;
    const uint64_t want = std::max(est, out->src.n + out->src.n / 2);
    GB_TRY(grow(out->src, m + lines, want, m, s));
    GB_TRY(grow(out->dst, m + lines, want, m, s));
    if (want_value) {
      GB_TRY(grow(out->w, m + lines, want, m, s));
      const uint64_t declined = text.host[1];
      GB_TRY(grow(dec_off, declined + lines, 2 * (declined + lines), declined, s));
      GB_TRY(grow(dec_edge, declined + lines, 2 * (declined + lines), declined, s));
    }
    k_load_parse_text<<<(unsigned)LineTiles::tiles(c), LOAD_BLOCK, 0, s>>>(
        reinterpret_cast<const uint4*>(c.dev), c.len, text.counts.p, m, c.off, want_value ? 1 : 0, out->src.p,
        out->dst.p, out->w.p, ctr.p, dec_off.p, dec_edge.p);
    GB_CUDA(cudaGetLastError());
    m += lines;
    return GB_OK;
  }
  gb_status finish(gb_load_info* info) {
    LoadCounters hc{};
    GB_CUDA(cudaMemcpyAsync(&hc, ctr.p, sizeof hc, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    GB_REQUIRE(hc.wide == 0, "edge list node id does not fit 32 bits");
    if (wcc) {
      info->edges = m;
      return wcc->finish_pairs(m);
    }
    // declined values: re-read each line and parse it with the host reader's own function
    if (hc.declined) {
      std::vector<uint64_t> off(hc.declined);
      std::vector<uint32_t> edge(hc.declined);
      GB_CUDA(cudaMemcpyAsync(off.data(), dec_off.p, hc.declined * 8ull, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaMemcpyAsync(edge.data(), dec_edge.p, hc.declined * 4ull, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      std::vector<float> val(hc.declined);
      std::string line;
      for (uint64_t i = 0; i < hc.declined; ++i) {
        GB_TRY(f.read_line(off[i], 256, &line));
        uint64_t src, dst;
        gb::parse_line(line.data(), 0, line.size(), 1, &src, &dst, &val[i]);
      }
      DevBuf<float> dval;
      GB_TRY(dval.alloc(hc.declined));
      GB_CUDA(cudaMemcpyAsync(dval.p, val.data(), hc.declined * 4ull, cudaMemcpyHostToDevice, s));
      k_load_patch<<<grid_for(hc.declined, 256), 256, 0, s>>>(dec_edge.p, dval.p, hc.declined, out->w.p);
      GB_CUDA(cudaGetLastError());
      GB_CUDA(cudaStreamSynchronize(s));
      info->h2d_bytes += hc.declined * 4ull;
    }
    out->m = m;
    out->n = 0;  // max id + 1
    info->edges = m;
    info->fallback_lines = hc.declined;
    return GB_OK;
  }
};

// DotGraph files after the header h, which the host has read.  The arrays are the caller's, NULL where they are
// not wanted or the file cannot hold the lines h declares (dot_fits).
struct DotGraphDecoder {
  cudaStream_t s;
  const DotHeader& h;
  uint32_t *labels, *src, *dst;
  WccSink* wcc = nullptr;  // instead of the arrays (labels not kept)
  LineTiles text;
  DevBuf<unsigned long long> first_error;  // line << 3 | code of the first bad line
  uint64_t line = 0;  // lines so far, the header included

  gb_status begin() {
    GB_TRY(text.begin());
    GB_TRY(first_error.alloc(1));
    GB_CUDA(cudaMemsetAsync(first_error.p, 0xFF, 8, s));
    if (wcc) GB_TRY(wcc->start(s, 0));
    return GB_OK;
  }
  gb_status stage(const Chunk& c, DeviceStaging& st) {
    if (wcc) GB_TRY(wcc->staging(c, st.sp.copy));
    return text.stage(c, st);
  }
  gb_status before(const Chunk& c) { return text.count(c, s); }
  gb_status after(const Chunk& c) {
    GB_CUDA(cudaStreamSynchronize(s));
    if (wcc) {
      // the chunk's edge lines N + 1 + e, e in [e0, e1), go to the pairs; a bad line leaves its pair (0, 0)
      const uint64_t first_edge_line = (uint64_t)h.nodes + 1, lines = text.lines(c);
      const uint64_t a = std::max(line, first_edge_line), b = std::min(line + lines, first_edge_line + h.edges);
      const uint64_t e0 = a - first_edge_line, count = b > a ? b - a : 0;
      uint32_t *ps = nullptr, *pd = nullptr;
      if (count) {
        GB_TRY(wcc->scratch(count));
        GB_CUDA(cudaMemsetAsync(wcc->src.p, 0, count * 4, s));
        GB_CUDA(cudaMemsetAsync(wcc->dst.p, 0, count * 4, s));
        ps = wcc->src.p - e0;  // the kernel stores edge e at src[e]
        pd = wcc->dst.p - e0;
      }
      k_load_parse_dotgraph<<<(unsigned)LineTiles::tiles(c), LOAD_BLOCK, 0, s>>>(
          reinterpret_cast<const uint4*>(c.dev), c.len, text.counts.p, line, h.nodes, h.lines, nullptr, ps, pd,
          first_error.p);
      GB_CUDA(cudaGetLastError());
      line += lines;
      return wcc->link_pairs(count, nullptr);
    }
    k_load_parse_dotgraph<<<(unsigned)LineTiles::tiles(c), LOAD_BLOCK, 0, s>>>(
        reinterpret_cast<const uint4*>(c.dev), c.len, text.counts.p, line, h.nodes, h.lines, labels, src, dst,
        first_error.p);
    GB_CUDA(cudaGetLastError());
    line += text.lines(c);
    return GB_OK;
  }
  gb_status finish(gb_load_info* info) {
    unsigned long long first = 0;
    GB_CUDA(cudaMemcpyAsync(&first, first_error.p, 8, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    if (first != ~0ull) return dot_fail((uint32_t)(first & 7), (first >> 3) + 1, h, 0);
    if (line < h.lines) return dot_fail(DOT_MISSING, 0, h, line);
    info->edges = h.edges;
    if (wcc) return wcc->finish_pairs(h.edges);
    return GB_OK;
  }
};

// The CSR (or label) arrays a binary file's section fills.  Elements of `stride` bytes start at file byte `pos`
// with an id (or label) of `width` bytes; a u32 section without values (stride 4) is DMA'd straight into `ids`,
// the others are staged and split by k_bin_split.  first_wide: see k_bin_split (NULL: the `wide` flag).
// A section whose targets a WccSink links (link = its CSR) is always staged: its chunks are split into the sink's
// scratch and linked there.
struct BinSection {
  uint64_t pos = 0, count = 0;
  uint32_t stride = 0, width = 0;
  uint32_t* ids = nullptr;
  float* w = nullptr;
  unsigned int* first_wide = nullptr;
  int link = -1;
  bool direct() const { return stride == 4 && link < 0; }
  uint64_t end() const { return pos + count * stride; }
};

// check_loaded_csrs's verdicts on CSR c: its offsets' first and last entries and decreasing rows, then its targets
// >= n
static gb_status bin_csr_verdict(const BinLayout& l, unsigned c, uint32_t first, unsigned int bad_rows, uint32_t last,
                                 unsigned int bad_targets) {
  const char* what = bin_csr_name(l, c);
  GB_REQUIRE(first == 0, "%s offsets[0] must be 0", what);
  GB_TRY(require_monotone(what, bad_rows));
  GB_REQUIRE(last == l.entries, "%s offsets end at %u, not at its %llu entries", what, last,
             (unsigned long long)l.entries);
  return require_ids(what, bad_targets, l.n);
}
static gb_status bin_wide_verdict(unsigned int wide) {
  GB_REQUIRE(wide == 0, "binary graph file: an id or offset does not fit 32 bits");
  return GB_OK;
}

// the checks of gb_binary_decode on the device arrays: offsets[0] == 0, monotone, offsets[n] == entries, targets
// below n; `wide` is the flag of the narrowing kernel
static gb_status check_loaded_csrs(const BinLayout& l, DevCsr* const* csr, unsigned int* d_wide, cudaStream_t s) {
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
  GB_TRY(bin_wide_verdict(h[4]));
  for (unsigned c = 0; c < l.ncsr; ++c) GB_TRY(bin_csr_verdict(l, c, e[2 * c], h[2 * c + 1], e[2 * c + 1], h[2 * c]));
  return GB_OK;
}

// Binary graph files, into the CSR arrays of g (and its label array, for a labelled layout l).  A staged chunk
// carries at most 15 bytes of a cut element in front, and k_bin_split decodes the elements that end inside the
// chunk.  With a WccSink (g NULL, l directed without labels) the offsets go into the sink's CSRs and each chunk's
// targets into its scratch, where they are linked.
struct BinaryDecoder {
  cudaStream_t s;
  gb_graph* g;
  const BinLayout& l;
  bool want_value;
  WccSink* wcc = nullptr;
  std::vector<BinSection> secs;
  DevBuf<unsigned int> wide;        // an id or offset does not fit 32 bits
  DevBuf<unsigned int> label_wide;  // the smallest node whose 8-byte label does not fit 32 bits, or ~0
  std::string carry;                // bytes of the staged element that the next chunk completes

  gb_status begin() {
    if (l.label_bytes) {
      GB_TRY(g->labels.alloc(l.n));
      GB_TRY(label_wide.alloc(1));
      GB_CUDA(cudaMemsetAsync(label_wide.p, 0xFF, 4, s));
      BinSection sec;
      sec.pos = BIN_USIZE, sec.count = l.n, sec.stride = sec.width = l.label_bytes, sec.ids = g->labels.p;
      sec.first_wide = label_wide.p;
      secs.push_back(sec);
    }
    for (unsigned c = 0; c < l.ncsr; ++c) {
      DevCsr& d = *csr(c);
      d.len = l.entries;
      GB_TRY(d.off.alloc((size_t)l.n + 1));
      if (!wcc) {
        GB_TRY(d.tgt.alloc(l.entries, 8));
        GB_CUDA(cudaMemsetAsync(d.tgt.p + l.entries, 0, 8 * 4, s));
      }
      if (c == 0 && want_value) GB_TRY(d.w.alloc(l.entries, 8));  // the out-CSR or the undirected CSR; no in-CSR values
      BinSection o, t;
      o.pos = l.csr[c].off_pos, o.count = (uint64_t)l.n + 1, o.stride = o.width = l.id_bytes, o.ids = d.off.p;
      t.pos = l.csr[c].rec_pos, t.count = l.entries, t.stride = l.rec_bytes, t.width = l.id_bytes, t.ids = d.tgt.p;
      t.w = d.w.p;
      if (wcc) t.link = (int)c;
      secs.push_back(o);
      if (t.count) secs.push_back(t);
    }
    GB_TRY(wide.alloc(1));
    GB_CUDA(cudaMemsetAsync(wide.p, 0, 4, s));
    if (wcc) return wcc->start(s, l.n);
    return GB_OK;
  }
  DevCsr* csr(unsigned c) const { return wcc ? &wcc->csr[c] : c == 0 ? &g->out : &g->in; }
  gb_status stage(const Chunk& c, DeviceStaging& st) {
    if (wcc) GB_TRY(wcc->staging(c, st.sp.copy));
    bool staged = false;
    for (const BinSection& sec : secs) staged |= !sec.direct() && sec.pos < c.b && sec.end() > c.a;
    if (staged) GB_TRY(st.stage(c.k, carry.data(), carry.size(), c.b - c.a));
    for (const BinSection& sec : secs) {
      if (!sec.direct()) continue;
      const uint64_t x = std::max(c.a, sec.pos), y = std::min(c.b, sec.end());
      if (x >= y) continue;
      GB_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(sec.ids) + (x - sec.pos), c.data + (x - c.a), y - x,
                              cudaMemcpyHostToDevice, st.sp.copy));
      st.h2d += y - x;
    }
    carry.clear();
    for (const BinSection& sec : secs)
      if (!sec.direct() && sec.pos < c.b && sec.end() > c.b) {
        const uint64_t cut = (c.b - sec.pos) % sec.stride;  // bytes of the element that begins before b
        carry.assign(c.data + (c.b - c.a - cut), cut);
      }
    return GB_OK;
  }
  gb_status before(const Chunk&) { return GB_OK; }
  gb_status after(const Chunk& c) {
    for (const BinSection& sec : secs) {
      if (sec.direct() || sec.pos >= c.b || sec.end() <= c.a) continue;
      const uint64_t first = c.a > sec.pos ? (c.a - sec.pos) / sec.stride : 0;  // the first element that ends after a
      const uint64_t last = std::min(sec.count, (c.b - sec.pos) / sec.stride);   // elements that end by b
      if (last <= first) continue;
      if (sec.link >= 0) {
        // elements [first, last) as elements [0, last - first) of a section that starts `first` elements later
        GB_TRY(wcc->scratch(last - first, false));
        k_bin_split<<<grid_for(last - first, 256), 256, 0, s>>>(c.dev, c.off, sec.pos + first * sec.stride, sec.stride,
                                                               sec.width, 0, last - first, wcc->src.p, nullptr, wide.p,
                                                               nullptr);
        GB_CUDA(cudaGetLastError());
        GB_TRY(wcc->link_targets((unsigned)sec.link, l, first, last - first));
        continue;
      }
      k_bin_split<<<grid_for(last - first, 256), 256, 0, s>>>(c.dev, c.off, sec.pos, sec.stride, sec.width, first,
                                                             last - first, sec.ids, sec.w, wide.p, sec.first_wide);
      GB_CUDA(cudaGetLastError());
    }
    return GB_OK;
  }
  gb_status finish(gb_load_info* info) {
    if (l.label_bytes == 8) {  // the labels first, as gb_binary_decode_labeled checks them
      unsigned int first = 0;
      GB_CUDA(cudaMemcpyAsync(&first, label_wide.p, 4, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      if (first != 0xFFFFFFFFu) return bin_label_wide(first);
    }
    info->edges = l.kind == GB_KIND_DIRECTED ? l.entries : l.entries / 2;
    if (wcc) {  // check_loaded_csrs's verdicts, on the checks made along the way
      unsigned int h[3] = {0, 0, 0};
      GB_CUDA(cudaMemcpyAsync(h, wide.p, 4, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaMemcpyAsync(h + 1, wcc->bad.p, 8, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      GB_TRY(bin_wide_verdict(h[0]));
      for (unsigned c = 0; c < l.ncsr; ++c) {
        GB_TRY(wcc->check_offsets(c, l.n));
        GB_TRY(bin_csr_verdict(l, c, wcc->off_first[c], wcc->off_bad[c], wcc->off_last[c], h[1 + c]));
      }
      return wcc->finish();
    }
    DevCsr* csr[2] = {&g->out, &g->in};
    GB_TRY(check_loaded_csrs(l, csr, wide.p, s));
    return GB_OK;
  }
};

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
  else if (want_value)
    GB_TRY(gb_graph_from_weighted_edges_u32(device, src.data(), dst.data(), w.data(), m, n, layout, graph));
  else
    GB_TRY(gb_graph_from_edges_u32(device, src.data(), dst.data(), m, n, layout, graph));
  info->edges = m;
  info->h2d_bytes = m * (want_value ? 12 : 8);
  return GB_OK;
}

// the edges of a Graph500 or edge-list file, parsed on the device into out
static gb_status stream_edges(int device, const InputFile& f, gb_file_format format, bool want_value,
                              EdgeArrays* out, gb_load_info* info) {
  if (format == GB_FORMAT_GRAPH500)
    return stream_file<Graph500Decoder>(device, f, 12 * (f.bytes / 12), 48, info, f.bytes / 12, out);
  return stream_file<EdgeListDecoder>(device, f, f.bytes, 1, info, f, want_value, out);
}

// a larger Graph500 or edge-list file (or any, with GB_LOAD_CHUNK_BYTES): parsed on the device, then
// gb_[di]graph_from_device_edges_u32's build
static gb_status load_edges_streamed(int device, gb_graph_kind kind, const InputFile& f, gb_file_format format,
                                     gb_layout layout, bool want_value, gb_graph** graph, gb_load_info* info) {
  EdgeArrays e;
  GB_TRY(stream_edges(device, f, format, want_value, &e, info));
  return graph_from_device_arrays(device, kind, e.src.p, e.dst.p, want_value ? e.w.p : nullptr, e.m, e.n, layout,
                                  nullptr, graph);
}

// A labelled graph has N nodes, one per label (csr.rs:554-562 asserts that every edge id is below it); an unlabelled
// one has max edge id + 1 (csr.rs:577-587), N only counting the node lines to skip.
static gb_status dot_require_nodes(const DotHeader& h, bool labeled) {
  GB_REQUIRE(!labeled || h.nodes > 0, "a labelled DotGraph needs at least one node line; the header declares N = 0");
  return GB_OK;
}
// A read without stores (dot_fits false) always meets a bad or missing line and fails first, so this guards a case
// that cannot arise: such a file never reaches the graph build.
static gb_status dot_require_fits(const DotHeader& h, bool fits) {
  GB_REQUIRE(fits, "DotGraph file is too short for the 1 + %u node + %u edge lines its header declares", h.nodes,
             h.edges);
  return GB_OK;
}

// a small DotGraph file: the host reader, then the upload of gb_[di]graph_from_edges[_labeled]_u32
static gb_status load_dotgraph_on_host(int device, gb_graph_kind kind, const InputFile& f, gb_layout layout,
                                       bool labeled, gb_graph** graph, gb_load_info* info) {
  std::unique_ptr<char[]> bytes;
  GB_TRY(f.read_all(&bytes));
  DotHeader h;
  GB_TRY(dot_read_header(bytes.get(), f.bytes, &h));
  const bool fits = dot_fits(h, f.bytes);
  std::vector<uint32_t> labels, src, dst;
  try {
    if (fits) labels.resize(labeled ? h.nodes : 0), src.resize(h.edges), dst.resize(h.edges);
  } catch (const std::bad_alloc&) {
    return fail(GB_ERR_OOM, "host allocation for %u labels and %u edges failed", h.nodes, h.edges);
  }
  GB_TRY(dot_read_host(bytes.get(), f.bytes, h, fits && labeled ? labels.data() : nullptr, fits ? src.data() : nullptr,
                       fits ? dst.data() : nullptr));
  GB_TRY(dot_require_fits(h, fits));
  GB_TRY(dot_require_nodes(h, labeled));
  if (labeled && kind == GB_KIND_DIRECTED)
    GB_TRY(gb_digraph_from_edges_labeled_u32(device, src.data(), dst.data(), h.edges, labels.data(), h.nodes, layout,
                                             graph));
  else if (labeled)
    GB_TRY(gb_graph_from_edges_labeled_u32(device, src.data(), dst.data(), h.edges, labels.data(), h.nodes, layout,
                                           graph));
  else if (kind == GB_KIND_DIRECTED)
    GB_TRY(gb_digraph_from_edges_u32(device, src.data(), dst.data(), nullptr, h.edges, 0, layout, graph));
  else
    GB_TRY(gb_graph_from_edges_u32(device, src.data(), dst.data(), h.edges, 0, layout, graph));
  info->edges = h.edges;
  info->h2d_bytes = 8ull * h.edges + (labeled ? 4ull * h.nodes : 0);
  return GB_OK;
}

// a larger DotGraph file (or any, with GB_LOAD_CHUNK_BYTES): the header on the host, the lines on the device
static gb_status load_dotgraph_streamed(int device, gb_graph_kind kind, const InputFile& f, gb_layout layout,
                                        bool labeled, gb_graph** graph, gb_load_info* info) {
  // the first line, as the host reader sees it in the whole file
  std::string head;
  GB_TRY(f.read_line(0, 4096, &head));
  DotHeader h;
  GB_TRY(dot_read_header(head.data(), head.size(), &h));
  const bool fits = dot_fits(h, f.bytes);
  DevBuf<uint32_t> src, dst, labels;
  if (fits) {
    GB_TRY(src.alloc(h.edges));
    GB_TRY(dst.alloc(h.edges));
    if (labeled) GB_TRY(labels.alloc(h.nodes));
  }
  GB_TRY(stream_file<DotGraphDecoder>(device, f, f.bytes, 1, info, h, labels.p, src.p, dst.p));
  GB_TRY(dot_require_fits(h, fits));
  GB_TRY(dot_require_nodes(h, labeled));
  GB_TRY(graph_from_device_arrays(device, kind, src.p, dst.p, nullptr, h.edges, labeled ? h.nodes : 0, layout, nullptr,
                                  graph));
  if (labeled) (*graph)->labels = std::move(labels);  // parsed on the device, so not part of h2d_bytes
  return GB_OK;
}

// a small binary file: gb_binary_decode (gb_binary_decode_labeled, for label_bytes != 0), then the upload of
// gb_[di]graph_from_csr_u32 and of the labels
static gb_status load_binary_on_host(int device, gb_graph_kind kind, const InputFile& f, bool want_value,
                                     uint32_t label_bytes, gb_graph** graph, gb_load_info* info) {
  std::unique_ptr<char[]> bytes;
  GB_TRY(f.read_all(&bytes));
  const uint64_t len = f.bytes;
  uint32_t n = 0;
  uint64_t m = 0;
  int has_values = 0;
  if (label_bytes)
    GB_TRY(gb_binary_decode_labeled(bytes.get(), len, kind, label_bytes, &n, &m, &has_values, nullptr, nullptr,
                                    nullptr, nullptr, nullptr, nullptr));
  else
    GB_TRY(gb_binary_decode(bytes.get(), len, kind, &n, &m, &has_values, nullptr, nullptr, nullptr, nullptr, nullptr));
  GB_REQUIRE(!want_value || has_values, "the binary graph file holds no edge values");
  const unsigned ncsr = kind == GB_KIND_DIRECTED ? 2 : 1;
  std::vector<uint32_t> off[2], tgt[2], labels(label_bytes ? n : 0);
  std::vector<float> w(want_value ? m : 0);
  for (unsigned c = 0; c < ncsr; ++c) off[c].resize((size_t)n + 1), tgt[c].resize(m);
  if (label_bytes)
    GB_TRY(gb_binary_decode_labeled(bytes.get(), len, kind, label_bytes, &n, &m, &has_values, labels.data(),
                                    off[0].data(), tgt[0].data(), nullptr, off[1].data(), tgt[1].data()));
  else
    GB_TRY(gb_binary_decode(bytes.get(), len, kind, &n, &m, &has_values, off[0].data(), tgt[0].data(),
                            want_value ? w.data() : nullptr, off[1].data(), tgt[1].data()));
  GraphPtr g;
  GB_TRY(new_graph(device, kind, n, &g));
  GB_TRY(upload_host_csr(g->stream, n, off[0].data(), tgt[0].data(), want_value ? w.data() : nullptr, &g->out,
                         kind == GB_KIND_DIRECTED ? "csr_out" : "csr"));
  if (kind == GB_KIND_DIRECTED)
    GB_TRY(upload_host_csr(g->stream, n, off[1].data(), tgt[1].data(), nullptr, &g->in, "csr_inc"));
  if (label_bytes) GB_TRY(attach_labels(g.get(), labels.data(), cudaMemcpyHostToDevice));
  *graph = g.release();
  info->edges = kind == GB_KIND_DIRECTED ? m : m / 2;
  info->h2d_bytes = ncsr * (((uint64_t)n + 1) * 4 + m * 4) + (want_value ? m * 4 : 0) + (label_bytes ? 4ull * n : 0);
  return GB_OK;
}

// a larger binary file (or any, with GB_LOAD_CHUNK_BYTES): the headers on the host, the sections streamed into the
// CSR arrays (and the label array, for label_bytes != 0)
static gb_status load_binary_streamed(int device, gb_graph_kind kind, const InputFile& f, bool want_value,
                                      uint32_t label_bytes, gb_graph** graph, gb_load_info* info) {
  BinLayout l;
  GB_TRY(bin_parse([&](uint64_t pos, void* dst, uint64_t n) { return pread_all(f.fd, static_cast<char*>(dst), n, pos); },
                   f.bytes, kind, &l, label_bytes));
  GB_REQUIRE(!want_value || l.values, "the binary graph file holds no edge values");
  GraphPtr g;
  GB_TRY(new_graph(device, kind, l.n, &g));
  GB_TRY(stream_file<BinaryDecoder>(device, f, f.bytes, 1, info, g.get(), l, want_value));
  *graph = g.release();
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
// interleaved on the device first: a weighted digraph's out- and in-CSR, a weighted undirected twin's one CSR).
// `labeled`: NodeValues<u32> in front of the CSRs, the count from host memory and the labels from device memory.
static gb_status serialize_graph(const gb_graph* g, const char* path, bool labeled) {
  GB_REQUIRE(g && path, "NULL argument");
  if (g->labels.p && !labeled)
    return fail(GB_ERR_UNSUPPORTED, "a labelled graph cannot be serialized: NodeValues payloads are not written");
  GB_REQUIRE(g->out.tgt.p != nullptr, "this handle holds no out targets (page-rank-only twin) and cannot be serialized");
  if (labeled && !g->labels.p)
    return fail(GB_ERR_UNSUPPORTED, "the graph has no node values to write (it was built without labels)");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  const bool values = !labeled && g->out.w.p != nullptr;  // a labelled twin's records carry no values
  const BinLayout l = bin_layout_u32(g->kind, g->n, g->out.len, values, labeled ? 4 : 0);
  const DevCsr* csr[2] = {&g->out, &g->in};
  DevBuf<float> in_w;
  if (values && g->kind == GB_KIND_DIRECTED) GB_TRY(in_csr_values(g, &in_w));
  struct Piece {
    uint64_t pos, len;
    const void* src;
    bool device;
  };
  std::vector<Piece> pieces;
  const uint64_t count = g->n;  // NodeValues' [usize n]
  if (labeled) {
    pieces.push_back({0, BIN_USIZE, &count, false});
    pieces.push_back({BIN_USIZE, (uint64_t)g->n * 4, g->labels.p, true});
  }
  std::string headers[2];
  DevBuf<uint2> records[2];
  for (unsigned c = 0; c < l.ncsr; ++c) {
    headers[c] = bin_header_bytes(l, c);
    pieces.push_back({c == 0 && !labeled ? 0 : l.csr[c].header, headers[c].size(), headers[c].data(), false});
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

// label_bytes: NV's width in a labelled binary file
static gb_status load_graph(int device, gb_graph_kind kind, const char* path, gb_file_format format,
                            gb_layout layout, int with_values, bool labeled, gb_graph** graph,
                            uint32_t label_bytes = 0) {
  GB_REQUIRE(graph != nullptr, "graph out-pointer is NULL");
  GB_REQUIRE(path != nullptr, "path is NULL");
  GB_REQUIRE(format == GB_FORMAT_GRAPH500 || format == GB_FORMAT_EDGE_LIST || format == GB_FORMAT_BINARY ||
                 format == GB_FORMAT_DOTGRAPH,
             "unknown file format %d", (int)format);
  GB_REQUIRE(!with_values || format == GB_FORMAT_EDGE_LIST || format == GB_FORMAT_BINARY,
             "only edge lists and binary files carry edge values");
  GB_TRY(check_layout(layout));
  if (labeled && format == GB_FORMAT_BINARY) GB_TRY(bin_check_label_bytes(label_bytes));
  else label_bytes = 0;
  GB_TRY(require_device(device));
  DeviceGuard guard(device);
  InputFile f;
  GB_TRY(f.open(path));
  gb_load_info info{};
  info.file_bytes = f.bytes;
  const bool on_host = env_chunk_bytes() == 0 && f.bytes < LOAD_DEVICE_MIN_BYTES;
  if (format == GB_FORMAT_DOTGRAPH) {
    if (on_host) GB_TRY(load_dotgraph_on_host(device, kind, f, layout, labeled, graph, &info));
    else GB_TRY(load_dotgraph_streamed(device, kind, f, layout, labeled, graph, &info));
  } else if (format == GB_FORMAT_BINARY) {
    if (on_host) GB_TRY(load_binary_on_host(device, kind, f, with_values != 0, label_bytes, graph, &info));
    else GB_TRY(load_binary_streamed(device, kind, f, with_values != 0, label_bytes, graph, &info));
  } else {
    if (on_host) GB_TRY(load_on_host(device, kind, f, format, layout, with_values != 0, graph, &info));
    else GB_TRY(load_edges_streamed(device, kind, f, format, layout, with_values != 0, graph, &info));
  }
  (*graph)->load = info;
  return GB_OK;
}

// The edges of a Graph500 or edge-list file on the device, for a graph that is not built by build_csr_device
// alone (the adjacency lists of adj_list.cu).  Always the streamed pipeline: the edge arrays it fills are what the
// caller keeps, so the host readers' upload would only add a copy.
gb_status load_edge_arrays(int device, const char* path, gb_file_format format, bool with_values, EdgeArrays* out) {
  GB_REQUIRE(path != nullptr, "path is NULL");
  GB_REQUIRE(format == GB_FORMAT_GRAPH500 || format == GB_FORMAT_EDGE_LIST,
             "adjacency lists load Graph500 and edge-list files, not format %d", (int)format);
  GB_REQUIRE(!with_values || format == GB_FORMAT_EDGE_LIST, "only edge lists carry edge values");
  GB_TRY(require_device(device));
  DeviceGuard guard(device);
  InputFile f;
  GB_TRY(f.open(path));
  out->info = gb_load_info{};
  out->info.file_bytes = f.bytes;
  return stream_edges(device, f, format, with_values, out, &out->info);
}

thread_local gb_wcc_file_stats wcc_file_last{};  // behind gb_wcc_file_info

// gb_wcc_file_u32: the file as load_graph(device, GB_KIND_DIRECTED, path, format, GB_LAYOUT_UNSORTED, 0) reads it
// on its streamed path, every decoded chunk handed to a WccSink.  The checks come in the load's order.
static gb_status wcc_file(int device, const char* path, gb_file_format format, const gb_wcc_config* cfg,
                          gb_components** out) {
  wcc_file_last = gb_wcc_file_stats{};
  GB_REQUIRE(out != nullptr, "components out-pointer is NULL");
  GB_REQUIRE(cfg != nullptr, "config is NULL");  // chunk_size / neighbor_rounds / sampling_size: labels unchanged
  GB_REQUIRE(path != nullptr, "path is NULL");
  GB_REQUIRE(format == GB_FORMAT_GRAPH500 || format == GB_FORMAT_EDGE_LIST || format == GB_FORMAT_BINARY ||
                 format == GB_FORMAT_DOTGRAPH,
             "unknown file format %d", (int)format);
  GB_TRY(require_device(device));
  DeviceGuard guard(device);
  InputFile f;
  GB_TRY(f.open(path));
  DevBufTally tally;
  WccSink sink;
  gb_load_info info{};
  info.file_bytes = f.bytes;
  if (format == GB_FORMAT_GRAPH500) {
    GB_TRY(stream_file<Graph500Decoder>(device, f, 12 * (f.bytes / 12), 48, &info, f.bytes / 12, nullptr, &sink));
  } else if (format == GB_FORMAT_EDGE_LIST) {
    GB_TRY(stream_file<EdgeListDecoder>(device, f, f.bytes, 1, &info, f, false, nullptr, &sink));
  } else if (format == GB_FORMAT_DOTGRAPH) {
    std::string head;
    GB_TRY(f.read_line(0, 4096, &head));
    DotHeader h;
    GB_TRY(dot_read_header(head.data(), head.size(), &h));
    GB_TRY(stream_file<DotGraphDecoder>(device, f, f.bytes, 1, &info, h, nullptr, nullptr, nullptr, &sink));
    GB_TRY(dot_require_fits(h, dot_fits(h, f.bytes)));
  } else {
    BinLayout l;
    GB_TRY(bin_parse([&](uint64_t pos, void* dst, uint64_t n) { return pread_all(f.fd, static_cast<char*>(dst), n, pos); },
                     f.bytes, GB_KIND_DIRECTED, &l));
    GB_TRY(stream_file<BinaryDecoder>(device, f, f.bytes, 1, &info, nullptr, l, false, &sink));
  }
  // an empty Graph500 or edge-list file streams no chunk (the load's build reports it)
  GB_REQUIRE(info.chunks > 0, "cannot infer node_count from an empty edge list");
  std::unique_ptr<gb_components> c(new (std::nothrow) gb_components());
  GB_REQUIRE(c != nullptr, "host allocation failed");
  c->device = device;
  c->n = (uint32_t)sink.n;
  c->labels = std::move(sink.parent);
  c->labels.untally();  // the handle outlives the call
  gb_wcc_file_stats& w = wcc_file_last;
  w.file_bytes = info.file_bytes;
  w.chunks = info.chunks;
  w.edges = info.edges;
  w.h2d_bytes = info.h2d_bytes;
  w.device_bytes = tally.peak;
  w.node_count = c->n;
  w.total_ms = sink.total_ms;
  *out = c.release();
  return GB_OK;
}

}  // namespace gb


extern "C" {

gb_status gb_digraph_load_u32(int device, const char* path, gb_file_format format, gb_layout layout,
                              int with_values, gb_graph** graph) {
  return gb::load_graph(device, GB_KIND_DIRECTED, path, format, layout, with_values, false, graph);
}

gb_status gb_graph_load_u32(int device, const char* path, gb_file_format format, gb_layout layout,
                            gb_graph** graph) {
  return gb::load_graph(device, GB_KIND_UNDIRECTED, path, format, layout, 0, false, graph);
}

gb_status gb_graph_load_weighted_u32(int device, const char* path, gb_file_format format, gb_layout layout,
                                     gb_graph** graph) {
  return gb::load_graph(device, GB_KIND_UNDIRECTED, path, format, layout, 1, false, graph);
}

gb_status gb_digraph_load_labeled_u32(int device, const char* path, gb_layout layout, gb_graph** graph) {
  return gb::load_graph(device, GB_KIND_DIRECTED, path, GB_FORMAT_DOTGRAPH, layout, 0, true, graph);
}

gb_status gb_graph_load_labeled_u32(int device, const char* path, gb_layout layout, gb_graph** graph) {
  return gb::load_graph(device, GB_KIND_UNDIRECTED, path, GB_FORMAT_DOTGRAPH, layout, 0, true, graph);
}

gb_status gb_digraph_load_labeled_binary_u32(int device, const char* path, gb_layout layout, uint32_t label_bytes,
                                             gb_graph** graph) {
  return gb::load_graph(device, GB_KIND_DIRECTED, path, GB_FORMAT_BINARY, layout, 0, true, graph, label_bytes);
}

gb_status gb_graph_load_labeled_binary_u32(int device, const char* path, gb_layout layout, uint32_t label_bytes,
                                           gb_graph** graph) {
  return gb::load_graph(device, GB_KIND_UNDIRECTED, path, GB_FORMAT_BINARY, layout, 0, true, graph, label_bytes);
}

gb_status gb_graph_serialize(const gb_graph* graph, const char* path) {
  return gb::serialize_graph(graph, path, false);
}

gb_status gb_graph_serialize_labeled(const gb_graph* graph, const char* path) {
  return gb::serialize_graph(graph, path, true);
}

gb_status gb_graph_load_info(const gb_graph* g, gb_load_info* info) {
  GB_REQUIRE(g && info, "NULL argument");
  *info = g->load;
  return GB_OK;
}

gb_status gb_wcc_file_u32(int device, const char* path, gb_file_format format, const gb_wcc_config* config,
                          gb_components** out) {
  return gb::wcc_file(device, path, format, config, out);
}

gb_status gb_components_node_count(const gb_components* c, uint32_t* node_count) {
  GB_REQUIRE(c && node_count, "NULL argument");
  *node_count = c->n;
  return GB_OK;
}

gb_status gb_components_copy(const gb_components* c, uint32_t* labels) {
  GB_REQUIRE(c && labels, "NULL argument");
  gb::DeviceGuard guard(c->device);
  GB_CUDA(cudaMemcpy(labels, c->labels.p, (size_t)c->n * 4, cudaMemcpyDeviceToHost));
  return GB_OK;
}

gb_status gb_components_free(gb_components* c) {
  if (!c) return GB_OK;
  gb::DeviceGuard guard(c->device);
  delete c;
  return GB_OK;
}

gb_status gb_wcc_file_info(gb_wcc_file_stats* info) {
  GB_REQUIRE(info != nullptr, "info is NULL");
  *info = gb::wcc_file_last;
  return GB_OK;
}

}  // extern "C"
