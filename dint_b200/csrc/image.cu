// image.cu -- state images of engines and clusters (dint_image_*, dint_cluster_image_*; the layout is in dint_b200.h):
// the host half of image.cuh's pack / unpack kernels, the file format and its checks.
#include <algorithm>
#include <cerrno>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include "host.cuh"
#include "image.cuh"

// ---- state images: the regions of snapshot_regions in a file, zero lines left out (image.cuh; layout in dint_b200.h) ----
static const char kImgMagic[8] = {'D', 'I', 'N', 'T', 'I', 'M', 'G', '1'};
static const char kCluMagic[8] = {'D', 'I', 'N', 'T', 'C', 'L', 'U', '1'};
constexpr uint32_t kImgVersion = 1;
constexpr uint32_t kImgMaxRegions = 32;
constexpr uint32_t kCfgKnownFlags = DINT_CFG_LOCK_HOLDER_KEYS | DINT_CFG_STORE_EBPF_MASK | DINT_CFG_TATP_EBPF | DINT_CFG_SMALLBANK_EBPF;
constexpr uint32_t kImgSets = 3;                     // blocks in flight: pack | copy | file
struct ImgHeader {
  char magic[8];
  uint32_t version, kind;
  dint_cfg cfg;
  uint32_t n_regions;
  uint64_t kv_capacity[kMaxTables];
  uint32_t tpool_cap, n_tables;
};
struct ImgRegion { uint32_t index, reserved; uint64_t bytes, blocks; };
struct CluManifest {
  char magic[8];
  uint32_t version, kind, shards, reserved;
  dint_cfg cfg;
  uint32_t reserved2;
};
static_assert(sizeof(dint_cfg) == 76 && sizeof(ImgHeader) == 144 && sizeof(ImgRegion) == 24 && sizeof(CluManifest) == 104,
              "the image layout of include/dint_b200.h");

static thread_local double g_img_times[4];           // dint_image_times: wall, kernels, copies, file (s)

struct ImgFd {
  int fd = -1;
  ~ImgFd() { if (fd >= 0) close(fd); }
};
static bool img_read(int fd, void* p, size_t n) {
  uint8_t* q = (uint8_t*)p;
  while (n) {
    const ssize_t k = read(fd, q, n);
    if (k < 0 && errno == EINTR) continue;
    if (k <= 0) return false;
    q += k;
    n -= (size_t)k;
  }
  return true;
}
static bool img_write(int fd, const void* p, size_t n) {
  const uint8_t* q = (const uint8_t*)p;
  while (n) {
    const ssize_t k = write(fd, q, n);
    if (k < 0 && errno == EINTR) continue;
    if (k <= 0) return false;
    q += k;
    n -= (size_t)k;
  }
  return true;
}
// writes `bytes` to path.tmp, fsyncs it and renames it to path: a crash never leaves a half file under the final name
// fsyncs the directory holding `path`, so that a rename or unlink in it is durable
static int img_sync_dir(const char* path) {
  std::string dir(path);
  const size_t slash = dir.find_last_of('/');
  dir = slash == std::string::npos ? std::string(".") : slash == 0 ? std::string("/") : dir.substr(0, slash);
  ImgFd d;
  d.fd = open(dir.c_str(), O_RDONLY | O_DIRECTORY);
  if (d.fd < 0 || fsync(d.fd) != 0) return set_errf(DINT_EIO, "image directory %s: fsync: %s", dir.c_str(), strerror(errno));
  return DINT_OK;
}
static int img_publish(const char* tmp, const char* path, int fd) {
  if (fsync(fd) != 0) return set_errf(DINT_EIO, "image %s: fsync: %s", tmp, strerror(errno));
  if (rename(tmp, path) != 0) return set_errf(DINT_EIO, "image %s: rename: %s", path, strerror(errno));
  return img_sync_dir(path);
}

// one block of a region: its device range
struct ImgBlock { uint32_t region; uint64_t index; uint8_t* p; uint64_t bytes; };
static std::vector<ImgBlock> img_blocks(const std::vector<std::pair<void*, size_t>>& regs) {
  std::vector<ImgBlock> out;
  for (uint32_t r = 0; r < regs.size(); r++)
    for (uint64_t off = 0, k = 0; off < regs[r].second; off += kImgBlock, k++)
      out.push_back({r, k, (uint8_t*)regs[r].first + off, std::min<uint64_t>(kImgBlock, regs[r].second - off)});
  return out;
}
// bytes a block stores for its lines: whole lines, except a partial last line, which keeps its in-range bytes
static uint64_t img_stored_bytes(uint64_t raw, const uint32_t* bitmap, uint64_t n_set) {
  const uint64_t L = img_lines(raw), rem = raw % kImgLine;
  uint64_t b = n_set * kImgLine;
  if (rem && ((bitmap[(L - 1) >> 5] >> ((L - 1) & 31)) & 1u)) b -= kImgLine - rem;
  return b;
}

// What both directions share: device scratch of the kernels, pinned host buffers, the ring's device staging, timing.
struct ImgPipe {
  dint_engine* e = nullptr;
  uint8_t* scratch = nullptr;                         // {ticket, tilebase[], sums, desc[], gdesc[]} of one launch
  uint32_t* bad = nullptr;                            // unpack verdict per block
  uint8_t* host[kImgSets] = {};
  unsigned long long* meta = nullptr;                 // pinned: {checksum, stored lines} per set (save)
  cudaEvent_t ev[kImgSets][4] = {};                   // kernel begin / end, copy begin / end
  size_t stage = 0;
  size_t ring_cap[kImgSets] = {};                     // the ring's staging before this call
  ~ImgPipe() {
    if (!e) return;
    cudaSetDevice(e->device);
    cudaDeviceSynchronize();
    // the 64 MiB staging buffers this call added to the ring go again: the ring allocates what a later call needs
    for (uint32_t b = 0; b < kImgSets; b++)
      if (e->ring.in[b].cap > ring_cap[b]) { cudaFree(e->ring.in[b].p); e->ring.in[b] = HostRing::Buf{}; }
    cudaFree(scratch);
    cudaFree(bad);
    for (uint8_t* h : host) if (h) cudaFreeHost(h);
    if (meta) cudaFreeHost(meta);
    for (auto& s : ev) for (cudaEvent_t x : s) if (x) cudaEventDestroy(x);
  }
  static constexpr size_t kTicket = 0, kSums = 16, kTilebase = 64, kDesc = kTilebase + 4 * kImgMaxTiles;
  static constexpr size_t kGdesc = kDesc + 8 * kImgMaxTiles, kBytes = kGdesc + 8 * (kImgMaxTiles / 32);
  int init(dint_engine* e_, uint64_t n_blocks) {
    e = e_;
    stage = img_words(kImgBlock) * 4 + kImgBlock;
    for (uint32_t b = 0; b < kImgSets; b++) ring_cap[b] = e->ring.in[b].cap;
    { int rc = ring_reserve(e, kImgSets, stage, 0, 0); if (rc) return rc; }
    CU(cudaMalloc(&scratch, kBytes));
    CU(cudaMalloc(&bad, 4 * (n_blocks ? n_blocks : 1)));
    CU(cudaMemsetAsync(bad, 0, 4 * (n_blocks ? n_blocks : 1), e->stream));
    for (uint32_t b = 0; b < kImgSets; b++) {
      CU(cudaHostAlloc((void**)&host[b], stage, cudaHostAllocDefault));
      for (cudaEvent_t& x : ev[b]) CU(cudaEventCreate(&x));
    }
    CU(cudaHostAlloc((void**)&meta, 2 * kImgSets * sizeof(unsigned long long), cudaHostAllocDefault));
    return DINT_OK;
  }
  ImgArgs args(const ImgBlock& k, uint8_t* staged) const {
    ImgArgs a{};
    a.raw = k.p;
    a.bytes = k.bytes;
    a.n_words = (uint32_t)img_words(k.bytes);
    a.n_tiles = (uint32_t)((img_lines(k.bytes) + kImgTileLines - 1) / kImgTileLines);
    a.bitmap = (uint32_t*)staged;
    a.lines = staged + (size_t)a.n_words * 4;
    a.ticket = (uint32_t*)(scratch + kTicket);
    a.sum = (unsigned long long*)(scratch + kSums);
    a.tilebase = (uint32_t*)(scratch + kTilebase);
    a.desc = (unsigned long long*)(scratch + kDesc);
    a.gdesc = (unsigned long long*)(scratch + kGdesc);
    return a;
  }
  // kernel and copy time of the block that used set b (its events are complete)
  int account(uint32_t b) {
    float k = 0, c = 0;
    CU(cudaEventElapsedTime(&k, ev[b][0], ev[b][1]));
    CU(cudaEventElapsedTime(&c, ev[b][2], ev[b][3]));
    g_img_times[1] += k * 1e-3;
    g_img_times[2] += c * 1e-3;
    return DINT_OK;
  }
};

static int image_save_impl(dint_engine* e, const char* path) {
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());                        // quiesce, as dint_snapshot_create
  std::vector<std::pair<void*, size_t>> regs;
  snapshot_regions(e, regs);
  for (auto& r : regs)
    if ((uintptr_t)r.first & 15) return set_err(DINT_EIO, "internal: a state region is not 16-byte aligned");
  const std::vector<ImgBlock> blocks = img_blocks(regs);
  ImgHeader h{};
  memcpy(h.magic, kImgMagic, 8);
  h.version = kImgVersion;
  h.kind = (uint32_t)e->kind;
  h.cfg = e->cfg;
  h.n_regions = (uint32_t)regs.size();
  h.n_tables = e->ctx.n_tables;
  for (uint32_t t = 0; t < e->ctx.n_tables; t++) h.kv_capacity[t] = e->ctx.tbl[t].cap_mask + 1;
  h.tpool_cap = e->ctx.tpool_cap;
  std::vector<ImgRegion> rec(regs.size());
  for (uint32_t r = 0; r < regs.size(); r++) rec[r] = {r, 0, regs[r].second, (regs[r].second + kImgBlock - 1) / kImgBlock};

  ImgPipe P;
  { int rc = P.init(e, blocks.size()); if (rc) return rc; }
  int grid = 0;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&grid, k_image_pack, kThreads, 0));
  grid *= e->sms;
  const std::string tmp = std::string(path) + ".tmp";
  ImgFd f;
  f.fd = open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
  if (f.fd < 0) return set_errf(DINT_EIO, "image %s: %s", tmp.c_str(), strerror(errno));
  auto fail = [&](int rc) { unlink(tmp.c_str()); return rc; };
  double t0 = now_s();
  if (!img_write(f.fd, &h, sizeof h) || !img_write(f.fd, rec.data(), rec.size() * sizeof(ImgRegion)))
    return fail(set_errf(DINT_EIO, "image %s: write: %s", tmp.c_str(), strerror(errno)));
  g_img_times[3] += now_s() - t0;
  HostRing& R = e->ring;
  const uint64_t N = blocks.size();
  std::vector<unsigned long long> sum(N), nset(N);
  // block j: packed on e->stream, copied to host set j % 3 on s_out, written to the file -- three blocks in flight
  for (uint64_t j = 0; j < N + 2; j++) {
    if (j < N) {
      const uint32_t b = (uint32_t)(j % kImgSets);
      if (j >= kImgSets) CU(cudaStreamWaitEvent(e->stream, R.d2h[b], 0));     // the set's previous block has left
      CU(cudaMemsetAsync(P.scratch, 0, ImgPipe::kBytes, e->stream));
      const ImgArgs a = P.args(blocks[j], R.in[b].p);
      CU(cudaEventRecord(P.ev[b][0], e->stream));
      k_image_pack<<<grid < (int)a.n_tiles ? grid : (int)a.n_tiles, kThreads, 0, e->stream>>>(a);
      CU(cudaGetLastError());
      CU(cudaEventRecord(P.ev[b][1], e->stream));
      e->stats.kernel_launches++;
      CU(cudaMemcpyAsync(P.meta + 2 * b, a.sum, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
      CU(cudaEventRecord(R.ready[b], e->stream));
    }
    if (j >= 1 && j - 1 < N) {
      const uint64_t k = j - 1;
      const uint32_t b = (uint32_t)(k % kImgSets);
      CU(cudaEventSynchronize(R.ready[b]));
      sum[k] = P.meta[2 * b];
      nset[k] = P.meta[2 * b + 1];
      CU(cudaStreamWaitEvent(R.s_out, R.ready[b], 0));
      CU(cudaEventRecord(P.ev[b][2], R.s_out));
      CU(cudaMemcpyAsync(P.host[b], R.in[b].p, img_words(blocks[k].bytes) * 4 + nset[k] * kImgLine, cudaMemcpyDeviceToHost, R.s_out));
      CU(cudaEventRecord(P.ev[b][3], R.s_out));
      CU(cudaEventRecord(R.d2h[b], R.s_out));
    }
    if (j >= 2) {
      const uint64_t k = j - 2;
      const uint32_t b = (uint32_t)(k % kImgSets);
      CU(cudaEventSynchronize(R.d2h[b]));
      { int rc = P.account(b); if (rc) return fail(rc); }
      const uint64_t words = img_words(blocks[k].bytes);
      const uint64_t bytes = words * 4 + img_stored_bytes(blocks[k].bytes, (const uint32_t*)P.host[b], nset[k]);
      t0 = now_s();
      if (!img_write(f.fd, P.host[b], bytes) || !img_write(f.fd, &sum[k], 8))
        return fail(set_errf(DINT_EIO, "image %s: write: %s", tmp.c_str(), strerror(errno)));
      g_img_times[3] += now_s() - t0;
    }
  }
  t0 = now_s();
  int rc = img_publish(tmp.c_str(), path, f.fd);
  g_img_times[3] += now_s() - t0;
  return rc ? fail(rc) : DINT_OK;
}

// Reads and checks an image's header and region table; touches no CUDA state.
static int image_read_header(int fd, const char* path, ImgHeader& h, std::vector<ImgRegion>& rec) {
  if (!img_read(fd, &h, sizeof h)) return set_errf(DINT_EIO, "image %s: truncated header", path);
  if (memcmp(h.magic, kImgMagic, 8) != 0) return set_errf(DINT_EINVAL, "image %s: bad magic (not a dint_b200 state image)", path);
  if (h.version != kImgVersion) return set_errf(DINT_EINVAL, "image %s: format version %u, this build reads %u", path, h.version, kImgVersion);
  if (h.kind >= DINT_NUM_KINDS) return set_errf(DINT_EINVAL, "image %s: unknown kind %u", path, h.kind);
  if (h.cfg.flags & ~kCfgKnownFlags) return set_errf(DINT_EINVAL, "image %s: unknown option flags 0x%x", path, h.cfg.flags & ~kCfgKnownFlags);
  if (h.n_regions > kImgMaxRegions || h.n_tables > kMaxTables) return set_errf(DINT_EINVAL, "image %s: %u regions, %u tables", path, h.n_regions, h.n_tables);
  for (uint32_t t = 0; t < h.n_tables; t++)
    if (h.kv_capacity[t] < 2 || h.kv_capacity[t] > (1ULL << 34) || (h.kv_capacity[t] & (h.kv_capacity[t] - 1)))
      return set_errf(DINT_EINVAL, "image %s: table %u has capacity %llu", path, t, (unsigned long long)h.kv_capacity[t]);
  rec.resize(h.n_regions);
  if (!img_read(fd, rec.data(), rec.size() * sizeof(ImgRegion))) return set_errf(DINT_EIO, "image %s: truncated region table", path);
  for (uint32_t r = 0; r < h.n_regions; r++)
    if (rec[r].index != r || rec[r].blocks != (rec[r].bytes + kImgBlock - 1) / kImgBlock)
      return set_errf(DINT_EINVAL, "image %s: region %u: bad record", path, r);
  return DINT_OK;
}

// want: the configuration a cluster gives this shard (the image must hold the same one; its chunk is the cluster's)
int image_open_impl(const char* path, int device, const dint_cfg* want, dint_engine** out) {
  *out = nullptr;
  ImgFd f;
  f.fd = open(path, O_RDONLY);
  if (f.fd < 0) return set_errf(DINT_EIO, "image %s: %s", path, strerror(errno));
  ImgHeader h;
  std::vector<ImgRegion> rec;
  double t0 = now_s();
  { int rc = image_read_header(f.fd, path, h, rec); if (rc) return rc; }
  g_img_times[3] += now_s() - t0;
  dint_cfg cfg = h.cfg;
  for (uint32_t t = 0; t < h.n_tables; t++) {
    uint32_t lg = 0;
    while ((1ULL << lg) < h.kv_capacity[t]) lg++;
    cfg.kv_capacity_log2[t] = lg;                   // (a tatp engine with the eBPF tier keeps its unused tables at 2^10)
  }
  if (want) {
    dint_cfg a = h.cfg, b = *want;
    a.chunk = b.chunk = 0;
    memset(a.kv_capacity_log2, 0, sizeof a.kv_capacity_log2);
    memset(b.kv_capacity_log2, 0, sizeof b.kv_capacity_log2);
    if (memcmp(&a, &b, sizeof a) != 0) return set_errf(DINT_EINVAL, "image %s: its configuration is not this shard's", path);
    cfg.chunk = want->chunk;
  }
  dint_engine* e = nullptr;
  { int rc = dint_create((int)h.kind, &cfg, device, &e); if (rc) return rc; }
  EngineOwner own{e};
  std::vector<std::pair<void*, size_t>> regs;
  snapshot_regions(e, regs);
  if (regs.size() != h.n_regions || e->ctx.tpool_cap != h.tpool_cap)
    return set_errf(DINT_EINVAL, "image %s: %u regions, this build lays the engine out in %u", path, h.n_regions, (uint32_t)regs.size());
  for (uint32_t r = 0; r < regs.size(); r++)
    if (regs[r].second != rec[r].bytes)
      return set_errf(DINT_EINVAL, "image %s: region %u holds %llu bytes, this build lays out %llu", path, r,
                      (unsigned long long)rec[r].bytes, (unsigned long long)regs[r].second);
  const std::vector<ImgBlock> blocks = img_blocks(regs);
  const uint64_t N = blocks.size();
  ImgPipe P;
  { int rc = P.init(e, N); if (rc) return rc; }
  int grid = 0;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&grid, k_image_unpack, kThreads, 0));
  grid *= e->sms;
  HostRing& R = e->ring;
  // block j: read into host set j % 3, copied to the device on s_in, checked and unpacked on e->stream
  for (uint64_t j = 0; j < N; j++) {
    const uint32_t b = (uint32_t)(j % kImgSets);
    const ImgBlock& k = blocks[j];
    if (j >= kImgSets) {                                // the set's previous block is unpacked
      CU(cudaEventSynchronize(R.released[b]));
      int rc = P.account(b);
      if (rc) return rc;
    }
    const uint64_t words = img_words(k.bytes);
    uint32_t* bm = (uint32_t*)P.host[b];
    uint8_t* lines = P.host[b] + words * 4;
    unsigned long long expect = 0;
    t0 = now_s();
    if (!img_read(f.fd, bm, words * 4)) return set_errf(DINT_EIO, "image %s: region %u block %llu: short read", path, k.region, (unsigned long long)k.index);
    uint64_t n_set = 0;
    for (uint64_t w = 0; w < words; w++) n_set += (uint64_t)__builtin_popcount(bm[w]);
    if (n_set > img_lines(k.bytes)) return set_errf(DINT_EIO, "image %s: region %u block %llu: checksum mismatch (bitmap)", path, k.region, (unsigned long long)k.index);
    const uint64_t stored = img_stored_bytes(k.bytes, bm, n_set);
    if (!img_read(f.fd, lines, stored) || !img_read(f.fd, &expect, 8))
      return set_errf(DINT_EIO, "image %s: region %u block %llu: short read", path, k.region, (unsigned long long)k.index);
    memset(lines + stored, 0, n_set * kImgLine - stored);   // a partial last line is hashed and staged zero-padded
    g_img_times[3] += now_s() - t0;
    if (j >= kImgSets) CU(cudaStreamWaitEvent(R.s_in, R.released[b], 0));
    CU(cudaEventRecord(P.ev[b][2], R.s_in));
    CU(cudaMemcpyAsync(R.in[b].p, P.host[b], words * 4 + n_set * kImgLine, cudaMemcpyHostToDevice, R.s_in));
    CU(cudaEventRecord(P.ev[b][3], R.s_in));
    CU(cudaEventRecord(R.h2d[b], R.s_in));
    CU(cudaStreamWaitEvent(e->stream, R.h2d[b], 0));
    CU(cudaMemsetAsync(P.scratch, 0, ImgPipe::kBytes, e->stream));
    ImgArgs a = P.args(k, R.in[b].p);
    a.expect = expect;
    a.bad = P.bad + j;
    CU(cudaEventRecord(P.ev[b][0], e->stream));
    CU(launch_ex(e, k_image_unpack, grid, kThreads, 0, e->stream, true, a));
    CU(cudaEventRecord(P.ev[b][1], e->stream));
    CU(cudaEventRecord(R.released[b], e->stream));
    e->stats.kernel_launches++;
  }
  {
    uint8_t extra;
    if (read(f.fd, &extra, 1) != 0) return set_errf(DINT_EINVAL, "image %s: bytes after the last block", path);
  }
  CU(cudaStreamSynchronize(e->stream));
  for (uint64_t j = N > kImgSets ? N - kImgSets : 0; j < N; j++) { int rc = P.account((uint32_t)(j % kImgSets)); if (rc) return rc; }
  std::vector<uint32_t> bad(N);
  if (N) CU(cudaMemcpy(bad.data(), P.bad, 4 * N, cudaMemcpyDeviceToHost));
  for (uint64_t j = 0; j < N; j++)
    if (bad[j]) return set_errf(DINT_EIO, "image %s: region %u block %llu: checksum mismatch", path, blocks[j].region, (unsigned long long)blocks[j].index);
  { int rc = engine_ready(e); if (rc) return rc; }
  own.e = nullptr;
  *out = e;
  return DINT_OK;
}

std::string img_shard_path(const char* dir, uint32_t r) { return std::string(dir) + "/shard-" + std::to_string(r) + ".img"; }
static std::string img_manifest_path(const char* dir) { return std::string(dir) + "/manifest"; }

extern "C" {

int dint_image_save(dint_engine* e, const char* path) {
  if (!e || !path) return set_err(DINT_EINVAL, "null argument");
  for (double& t : g_img_times) t = 0;
  const double t0 = now_s();
  const int rc = image_save_impl(e, path);
  g_img_times[0] = now_s() - t0;
  return rc;
}

int dint_image_open(const char* path, int device, dint_engine** out) {
  if (!path || !out) return set_err(DINT_EINVAL, "null argument");
  *out = nullptr;
  for (double& t : g_img_times) t = 0;
  const double t0 = now_s();
  const int rc = image_open_impl(path, device, nullptr, out);
  g_img_times[0] = now_s() - t0;
  return rc;
}

int dint_image_times(double out[4]) {
  if (!out) return DINT_EINVAL;
  for (int i = 0; i < 4; i++) out[i] = g_img_times[i];
  return DINT_OK;
}

int dint_cluster_image_save(dint_cluster* cl, const char* dir) {
  if (!cl || !dir) return set_err(DINT_EINVAL, "null argument");
  for (double& t : g_img_times) t = 0;
  const double t0 = now_s();
  if (mkdir(dir, 0755) != 0 && errno != EEXIST) return set_errf(DINT_EIO, "image directory %s: %s", dir, strerror(errno));
  // a manifest names shard images of one moment: an earlier one goes (durably) before the first shard is replaced, so a
  // save that stops part-way leaves a directory that opens as nothing rather than as shards of two moments
  const std::string manifest = img_manifest_path(dir);
  if (unlink(manifest.c_str()) != 0 && errno != ENOENT) return set_errf(DINT_EIO, "image %s: unlink: %s", manifest.c_str(), strerror(errno));
  { int rc = img_sync_dir(manifest.c_str()); if (rc) return rc; }
  int rc = DINT_OK;
  for (uint32_t r = 0; r < cl->G && rc == DINT_OK; r++) rc = image_save_impl(cl->eng[r], img_shard_path(dir, r).c_str());
  if (rc == DINT_OK) {                                  // the manifest last: a directory with one names complete shard images
    CluManifest m{};
    memcpy(m.magic, kCluMagic, 8);
    m.version = kImgVersion;
    m.kind = (uint32_t)cl->kind;
    m.shards = cl->G;
    m.cfg = cl->base;
    const std::string path = img_manifest_path(dir), tmp = path + ".tmp";
    ImgFd f;
    f.fd = open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (f.fd < 0 || !img_write(f.fd, &m, sizeof m)) rc = set_errf(DINT_EIO, "image %s: %s", tmp.c_str(), strerror(errno));
    else rc = img_publish(tmp.c_str(), path.c_str(), f.fd);
  }
  g_img_times[0] = now_s() - t0;
  return rc;
}

// dint_cluster_image_open; with `rebuilt` dint_cluster_image_open_rebuild
static int cluster_image_open(const char* dir, int n_gpus, const int* devices, uint64_t max_batch, uint32_t* rebuilt,
                              dint_cluster** out) {
  if (!dir || !out) return set_err(DINT_EINVAL, "null argument");
  *out = nullptr;
  if (rebuilt) *rebuilt = 0;
  for (double& t : g_img_times) t = 0;
  const double t0 = now_s();
  const std::string path = img_manifest_path(dir);
  CluManifest m;
  {
    ImgFd f;
    f.fd = open(path.c_str(), O_RDONLY);
    if (f.fd < 0) return set_errf(DINT_EIO, "image %s: %s", path.c_str(), strerror(errno));
    if (!img_read(f.fd, &m, sizeof m)) return set_errf(DINT_EIO, "image %s: truncated manifest", path.c_str());
  }
  if (memcmp(m.magic, kCluMagic, 8) != 0) return set_errf(DINT_EINVAL, "image %s: bad magic (not a dint_b200 cluster manifest)", path.c_str());
  if (m.version != kImgVersion) return set_errf(DINT_EINVAL, "image %s: format version %u, this build reads %u", path.c_str(), m.version, kImgVersion);
  if (m.kind >= DINT_NUM_KINDS || (m.cfg.flags & ~kCfgKnownFlags)) return set_errf(DINT_EINVAL, "image %s: unknown kind or option flags", path.c_str());
  if ((uint32_t)n_gpus != m.shards) return set_errf(DINT_EINVAL, "image %s: %u shards, not %d", path.c_str(), m.shards, n_gpus);
  uint32_t missing = 0;
  for (uint32_t r = 0; r < m.shards; r++) {
    struct stat st;
    if (stat(img_shard_path(dir, r).c_str(), &st) == 0) continue;
    if (!rebuilt) return set_errf(DINT_EIO, "image %s: %s", img_shard_path(dir, r).c_str(), strerror(errno));
    missing |= 1u << r;
  }
  if (missing && rebuild_check((int)m.kind, m.cfg, m.shards, missing))   // refused before any CUDA call
    return set_errf(DINT_EIO, "image %s: shard image(s) %s missing and cannot be rebuilt: %s", dir, mask_names(missing).c_str(),
                    g_last_error.c_str());
  if (rebuilt) { for (double& t : g_rebuild_times) t = 0; *rebuilt = missing; }
  const int rc = cluster_make((int)m.kind, &m.cfg, n_gpus, devices, max_batch, dir, nullptr, rebuilt, out);
  if (rc && rebuilt) *rebuilt = 0;
  g_img_times[0] = now_s() - t0;
  if (rebuilt) g_rebuild_times[0] = g_img_times[0];
  return rc;
}

int dint_cluster_image_open(const char* dir, int n_gpus, const int* devices, uint64_t max_batch, dint_cluster** out) {
  return cluster_image_open(dir, n_gpus, devices, max_batch, nullptr, out);
}

int dint_cluster_image_open_rebuild(const char* dir, int n_gpus, const int* devices, uint64_t max_batch, uint32_t* rebuilt_mask,
                                    dint_cluster** out) {
  if (!rebuilt_mask) return set_err(DINT_EINVAL, "null argument");
  return cluster_image_open(dir, n_gpus, devices, max_batch, rebuilt_mask, out);
}

}  // extern "C"
