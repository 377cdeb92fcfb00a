// dint_udp_server -- the reference's UDP server, with the per-datagram handler replaced by the batched engine.
//
// What it replaces: `<bench>/udp/server*.cc` of the reference: N pinned threads, each
// `recvfrom -> fasthash64 -> switch(type) -> sendto` on its own SO_REUSEPORT socket (lock_fasst/udp/server.cc:40-119,
// tatp/udp/server_shard.cc:213-260).  Same wire protocol (one packed `struct message` per datagram, the reply is
// the request buffer mutated and sent back to the source address), same default port (20230), so the reference's
// clients (`client_udp*`) talk to it unchanged.
//
// Shape: R socket threads (SO_REUSEPORT, like the reference's N threads) each alternate
//     recvmmsg (a batch) -> hand the batch to an engine thread -> sendmmsg (the replies),
// and TWO engine threads take turns: each gathers whatever batches are ready, in socket order, into its own pinned
// array, makes ONE submit call for all of them (H2D, kernels, D2H inside) and hands every socket thread its slice of
// the replies -- while one gathering is on the GPU the other thread collects and copies the next one.
// Order: datagrams of one socket (one client 4-tuple always hashes to the same socket) keep their arrival
// order inside the array, and request i of a submit sees the effects of every earlier one -- what ONE reference
// thread would have produced for that arrival order.  (Across sockets the reference has no order either.)
//
// --gpus N: the key space is served by N GPUs of this box through the C-level cluster API (dint_cluster_*): lock
// servers and store route every request to the GPU that owns its slot; tatp / smallbank keep the reference's
// deployment of one `server_shard` per address -- here shard i listens on port P + i and the port a datagram arrives
// on is the shard the client chose (tatp/caladan/client_udp_shard.cc:187: `key % kNumServers` picks the address).
//
// Caladan clients (lock_2pl/caladan/client_caladan.cc:248-271) first ask the server for data ports: a 4-byte
// `net_req{int nports}` datagram on the well-known port is answered with `net_resp{int nports; uint16_t ports[]}` after
// the server has opened that many fresh sockets (lock_2pl/caladan/proto.h:32-39, server.cc:107-146).  No wire message
// is 4 bytes long, so the same port serves both: a 4-byte datagram is a control request, everything else is data.
//
// Host C++ above the C ABI only (include/dint_b200.h): no CUDA here, no oracle, no CPU fallback -- without a
// GPU dint_create() fails and the server exits.
//
// usage: dint_udp_server <lock_2pl|lock_fasst|log_server|store|tatp|smallbank> [--port P] [--bind A.B.C.D]
//                        [--sockets R] [--batch N] [--device D] [--gpus G [--devices a,b,..]] [--shard-id I --shards G]
//                        [--linger-us U] [--populate N] [--mon-port 20231] [--lock-holder-keys]
//                        [--store-ebpf wb-bloom|wb|wt] [--tatp-ebpf] [--smallbank-ebpf] [--image-in PATH [--rebuild-lost]]
//                        [--image-out PATH]
//
// --lock-holder-keys (tatp): DINT_CFG_LOCK_HOLDER_KEYS -- a refused kAcquireLock is answered kRejectLockSameKey (28) when
// the lock is held for the same key and kRejectLock (8) when another key shares the slot, as the reference's eBPF lock
// server answers (tatp/ebpf/lock_kern.c:289-298); a client that speaks tatp/caladan/proto.h counts the two apart.
//
// --store-ebpf V (store): DINT_CFG_STORE_EBPF_* -- answer as the reference's eBPF store server (store/ebpf/store_kern.c,
// store_wb_kern.c, store_wt_kern.c for V = wb-bloom, wb, wt), with its per-bucket cache sets in front of the table; the
// server starts empty and --populate N serves the eBPF client's kInsert stream for N subscribers
// (store/caladan/client_ebpf.cc:137-180).
//
// --tatp-ebpf (tatp): DINT_CFG_TATP_EBPF -- answer as the reference's eBPF TATP shard server (tatp/ebpf/shard_kern.c;
// with --lock-holder-keys, lock_kern.c), with its per-bucket cache sets and bloom words in front of chained tables; the
// server starts empty and --populate N serves the eBPF client's insert stream for N subscribers
// (tatp/caladan/client_ebpf_shard.cc:96-339).  Every reply is one 55-byte struct message: the reference sends a
// kCommitBck that missed its cache back as the 108-byte ext_message (shard_kern.c:1231), whose first 55 bytes these are.
//
// --smallbank-ebpf (smallbank): DINT_CFG_SMALLBANK_EBPF -- answer as the reference's eBPF SmallBank shard server
// (smallbank/ebpf/shard_kern.c), with its per-bucket write-back cache sets in front of the account tables; --populate N
// inserts N accounts and then serves the eBPF client's warm-up stream for them (smallbank/caladan/
// client_ebpf_shard.cc:88-169), so the cache starts as the reference's clients leave it.
//
// --image-in PATH: start from a state image (include/dint_b200.h, "State images") instead of populating: a file written by
// dint_image_save, or with --gpus G > 1 a directory written by dint_cluster_image_save.  Its kind and option flags must
// be the command line's, and for tatp / smallbank with --shards G --shard-id I it must be shard I of G, else the server
// exits with 2.  --rebuild-lost (tatp / smallbank with --gpus G > 1): a shard image of the --image-in directory that is
// missing, short or corrupt is rebuilt from the other shards' replicas (dint_cluster_image_open_rebuild) and the server
// names the shards it rebuilt; without it such a directory stops start-up.  --image-out PATH: on SIGINT / SIGTERM, once the engine threads
// have stopped and the last replies are sent, write the state to PATH (the same file / directory forms); the exit code
// is 1 if that fails.
//
// --mon-port P: the reference servers' utilisation channel (tatp/udp/server_shard.cc:213-274: a thread samples the CPU
// time of the server's cores once a second, another answers any datagram on UDP :20231 with `struct {double ucores;
// double kcores;}`).  Here the two doubles are the user / kernel CPU cores this process used over the last second
// (getrusage) -- with the handler on the GPU that is what the host still spends on the sockets.
#include <arpa/inet.h>
#include <netinet/in.h>
#include <poll.h>
#include <signal.h>
#include <sys/resource.h>
#include <sys/socket.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

extern "C" {
#include "../../include/dint_b200.h"
}
// The state-image calls bind weakly: a library that serves requests without them (the CPU stand-in of the front-end's
// own tests) still loads; only --image-in / --image-out need them, and say so when they are missing.
#pragma weak dint_image_open
#pragma weak dint_image_save
#pragma weak dint_cluster_image_open
#pragma weak dint_cluster_image_save
#pragma weak dint_cluster_image_open_rebuild

namespace {

std::atomic<bool> g_stop{false};
void on_signal(int) { g_stop.store(true); }

// one socket thread's batch: filled by recvmmsg, answered in place, sent back with sendmmsg
struct Worker {
  std::vector<int> fds;                 // 1 socket (a listener) or the data sockets opened for one control request
  int group = 0;                        // --gpus with tatp / smallbank: the shard whose port these sockets serve
  bool control = false;                 // listens on a well-known port: 4-byte datagrams are control requests
  std::vector<uint8_t> buf;             // n * msg: requests in, replies out
  std::vector<mmsghdr> hdr;
  std::vector<iovec> iov;
  std::vector<sockaddr_in> peer;
  std::vector<int> from;                // fd index of every datagram
  int n = 0, dirty = 0;                 // dirty: headers the kernel wrote into during the last receive
  enum State { FILLING, READY, IN_FLIGHT, DONE } state = FILLING;   // guarded by the shared mutex
  uint64_t datagrams = 0, dropped = 0, controls = 0;
  std::thread th;
};

const char* const kKindNames[] = {"lock_2pl", "lock_fasst", "log_server", "store", "tatp", "smallbank"};
int kind_of(const std::string& s) {
  for (int k = 0; k < 6; k++)
    if (s == kKindNames[k]) return k;
  return -1;
}
const char* kind_name(uint32_t k) { return kKindNames[k]; }

int open_socket(const sockaddr_in& addr, bool reuseport) {
  int fd = socket(AF_INET, SOCK_DGRAM, 0);
  if (fd < 0) return -1;
  int one = 1, buf = 32 << 20;
  if (reuseport) setsockopt(fd, SOL_SOCKET, SO_REUSEPORT, &one, sizeof one);
  setsockopt(fd, SOL_SOCKET, SO_RCVBUF, &buf, sizeof buf);
  setsockopt(fd, SOL_SOCKET, SO_SNDBUF, &buf, sizeof buf);
  if (bind(fd, (const sockaddr*)&addr, sizeof addr) < 0) { close(fd); return -1; }
  return fd;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 2) {
    fprintf(stderr, "usage: %s <lock_2pl|lock_fasst|log_server|store|tatp|smallbank> [--port P] [--bind ADDR] [--sockets R] "
                    "[--batch N] [--device D] [--gpus G [--devices a,b,..]] [--shards G --shard-id I] [--linger-us U] [--populate N] [--lock-holder-keys] [--store-ebpf wb-bloom|wb|wt] [--tatp-ebpf] [--smallbank-ebpf] [--image-in PATH [--rebuild-lost]] [--image-out PATH]\n", argv[0]);
    return 2;
  }
  const int kind = kind_of(argv[1]);
  if (kind < 0) { fprintf(stderr, "unknown server kind '%s'\n", argv[1]); return 2; }
  int port = 20230, device = 0, linger_us = 50, gpus = 1, populate = -1, mon_port = 0;
  unsigned batch_max = 16384, shards = 1, shard_id = 0;
  unsigned n_sock = std::thread::hardware_concurrency() / 2;
  if (n_sock < 1) n_sock = 1;
  if (n_sock > 8) n_sock = 8;                         // the reference runs `server 8` (exp/run_lock_fasst.sh)
  std::string bind_addr = "0.0.0.0", image_in, image_out;
  std::vector<int> devices;
  bool holder_keys = false, tatp_ebpf = false, smallbank_ebpf = false, rebuild_lost = false;
  uint32_t store_ebpf = 0;
  for (int i = 2; i < argc; i += 2) {
    const std::string a = argv[i];
    if (a == "--lock-holder-keys") { holder_keys = true; i--; continue; }   // the three options without a value
    if (a == "--tatp-ebpf") { tatp_ebpf = true; i--; continue; }
    if (a == "--smallbank-ebpf") { smallbank_ebpf = true; i--; continue; }
    if (a == "--rebuild-lost") { rebuild_lost = true; i--; continue; }
    if (i + 1 >= argc) break;
    const char* v = argv[i + 1];
    if (a == "--port") port = atoi(v);
    else if (a == "--bind") bind_addr = v;
    else if (a == "--batch") batch_max = (unsigned)atoi(v);
    else if (a == "--sockets") n_sock = (unsigned)atoi(v);
    else if (a == "--device") device = atoi(v);
    else if (a == "--gpus") gpus = atoi(v);
    else if (a == "--devices") { for (const char* p = v; *p;) { devices.push_back(atoi(p)); while (*p && *p != ',') p++; if (*p) p++; } }
    else if (a == "--shards") shards = (unsigned)atoi(v);
    else if (a == "--shard-id") shard_id = (unsigned)atoi(v);
    else if (a == "--linger-us") linger_us = atoi(v);
    else if (a == "--populate") populate = atoi(v);
    else if (a == "--mon-port") mon_port = atoi(v);
    else if (a == "--image-in") image_in = v;
    else if (a == "--image-out") image_out = v;
    else if (a == "--store-ebpf") {
      const std::string w = v;
      if (w == "wb-bloom") store_ebpf = DINT_CFG_STORE_EBPF_WB_BLOOM;
      else if (w == "wb") store_ebpf = DINT_CFG_STORE_EBPF_WB;
      else if (w == "wt") store_ebpf = DINT_CFG_STORE_EBPF_WT;
      else { fprintf(stderr, "--store-ebpf takes wb-bloom, wb or wt\n"); return 2; }
    }
    else { fprintf(stderr, "unknown option %s\n", a.c_str()); return 2; }
  }
  if (batch_max < 1) batch_max = 1;
  if (n_sock < 1) n_sock = 1;
  if (n_sock > 64) n_sock = 64;
  if (gpus < 1 || gpus > 8 || (!devices.empty() && (int)devices.size() != gpus)) { fprintf(stderr, "bad --gpus / --devices\n"); return 2; }
  if (!image_in.empty() && populate >= 0) { fprintf(stderr, "--image-in and --populate exclude each other\n"); return 2; }
  if ((!image_in.empty() || !image_out.empty()) && !(dint_image_open && dint_image_save && dint_cluster_image_open && dint_cluster_image_save)) {
    fprintf(stderr, "dint_udp_server: this libdint_b200.so has no state images (--image-in / --image-out)\n");
    return 1;
  }
  const bool by_dst = kind == DINT_TATP || kind == DINT_SMALLBANK;
  if (rebuild_lost && (image_in.empty() || gpus < 2 || !by_dst)) {
    fprintf(stderr, "--rebuild-lost needs --image-in DIR with --gpus G > 1 and a tatp or smallbank server\n");
    return 2;
  }
  if (rebuild_lost && !dint_cluster_image_open_rebuild) {
    fprintf(stderr, "dint_udp_server: this libdint_b200.so cannot rebuild shards (--rebuild-lost)\n");
    return 1;
  }
  sockaddr_in srv{};
  srv.sin_family = AF_INET;
  if (inet_pton(AF_INET, bind_addr.c_str(), &srv.sin_addr) != 1) { fprintf(stderr, "bad --bind address\n"); return 2; }
  const uint32_t msg = dint_msg_size(kind);
  const int n_groups = (gpus > 1 && by_dst) ? gpus : 1;        // one well-known port per shard server

  // ---- engine: the state the reference keeps in its global arrays lives on the GPU(s) ----
  dint_cfg cfg;
  dint_default_cfg(kind, &cfg);                       // kLockHashSize, table sizes, ring length of the reference
  if (holder_keys) cfg.flags |= DINT_CFG_LOCK_HOLDER_KEYS;   // dint_create refuses it for a kind other than tatp
  cfg.flags |= store_ebpf;                                   // ... and this for a kind other than store
  if (tatp_ebpf) cfg.flags |= DINT_CFG_TATP_EBPF;            // ... and this for a kind other than tatp
  if (smallbank_ebpf) cfg.flags |= DINT_CFG_SMALLBANK_EBPF;  // ... and this for a kind other than smallbank
  if (populate >= 0) { cfg.subs_populate = (uint32_t)populate; cfg.accts_populate = (uint32_t)populate; }   // a prefix of the reference's population
  dint_engine* eng = nullptr;
  dint_cluster* cluster = nullptr;
  if (!image_in.empty()) {
    // the header's kind and dint_cfg (a state image: at byte 12 and 16; a cluster manifest: at byte 12 and 24)
    const bool dir = gpus > 1;
    FILE* f = fopen(dir ? (image_in + "/manifest").c_str() : image_in.c_str(), "rb");
    uint8_t hdr[104] = {0};
    const size_t got = f ? fread(hdr, 1, sizeof hdr, f) : 0;
    if (f) fclose(f);
    uint32_t img_kind = 0;
    dint_cfg img_cfg{};
    memcpy(&img_kind, hdr + 12, 4);
    memcpy(&img_cfg, hdr + (dir ? 24 : 16), sizeof img_cfg);
    if (got == sizeof hdr && ((int)img_kind != kind || img_cfg.flags != cfg.flags)) {
      fprintf(stderr, "dint_udp_server: %s holds a %s server with option flags 0x%x; the command line asks for %s with 0x%x\n",
              image_in.c_str(), img_kind < 6 ? kind_name(img_kind) : "unknown", img_cfg.flags, argv[1], cfg.flags);
      return 2;
    }
    // server_shard <id> of a G-shard deployment (--shards / --shard-id): the image must be that shard's (txn_shards 0 and
    // 1 both mean "every key")
    auto placement = [](uint32_t g) { return g > 1 ? g : 1u; };
    if (got == sizeof hdr && !dir && by_dst &&
        (placement(img_cfg.txn_shards) != placement(shards) || (placement(shards) > 1 && img_cfg.txn_shard_id != shard_id))) {
      fprintf(stderr, "dint_udp_server: %s holds shard %u of %u; the command line asks for shard %u of %u\n", image_in.c_str(),
              img_cfg.txn_shard_id, placement(img_cfg.txn_shards), shard_id, placement(shards));
      return 2;
    }
    uint32_t rebuilt = 0;
    const int* dv = devices.empty() ? nullptr : devices.data();
    const int rc = rebuild_lost ? dint_cluster_image_open_rebuild(image_in.c_str(), gpus, dv, 0, &rebuilt, &cluster)
                   : dir        ? dint_cluster_image_open(image_in.c_str(), gpus, dv, 0, &cluster)
                                : dint_image_open(image_in.c_str(), device, &eng);
    if (rc != DINT_OK) {
      fprintf(stderr, "dint_udp_server: opening the image failed: %s\n", dint_last_error());
      return 1;
    }
    if (rebuild_lost) {
      std::string names;
      for (int r = 0; r < gpus; r++)
        if ((rebuilt >> r) & 1u) names += (names.empty() ? "" : ", ") + std::to_string(r);
      fprintf(stderr, "dint_udp_server: rebuilt shard(s) {%s} of %s from their replicas\n", names.c_str(), image_in.c_str());
    }
  } else if (gpus > 1) {
    if (dint_cluster_create(kind, &cfg, gpus, devices.empty() ? nullptr : devices.data(), 0, &cluster) != DINT_OK ||
        dint_cluster_populate(cluster) != DINT_OK) {
      fprintf(stderr, "dint_udp_server: dint_cluster_create/populate failed: %s\n", dint_last_error());
      return 1;
    }
  } else {
    if (by_dst) {                                     // server_shard <id>: the CLIENT picks the shard; each holds its replicas
      cfg.txn_shards = shards;
      cfg.txn_shard_id = shard_id;
    }
    if (dint_create(kind, &cfg, device, &eng) != DINT_OK) {
      fprintf(stderr, "dint_udp_server: dint_create failed: %s\n", dint_last_error());
      return 1;
    }
    if (dint_populate(eng) != DINT_OK) {              // kvs_init + populate_* of the reference (no-op for lock / log)
      fprintf(stderr, "dint_udp_server: dint_populate failed: %s\n", dint_last_error());
      return 1;
    }
  }

  std::mutex mu;
  std::condition_variable cv_engine, cv_workers;
  std::vector<std::unique_ptr<Worker>> w;            // grows when control requests open data sockets (under mu)
  std::atomic<uint64_t> submits{0}, bad_batches{0};

  auto make_worker = [&](std::vector<int> fds, int group, bool control) {
    std::unique_ptr<Worker> x(new Worker());
    x->fds = std::move(fds);
    x->group = group;
    x->control = control;
    x->buf.resize((size_t)batch_max * msg);
    x->hdr.resize(batch_max);
    x->iov.resize(batch_max);
    x->peer.resize(batch_max);
    x->from.resize(batch_max);
    for (unsigned q = 0; q < batch_max; q++) {         // datagram q always lands in slot q of the batch buffer
      x->iov[q] = {x->buf.data() + (size_t)q * msg, msg};
      x->hdr[q].msg_hdr = {&x->peer[q], sizeof(sockaddr_in), &x->iov[q], 1, nullptr, 0, 0};
      x->hdr[q].msg_len = 0;
    }
    return x;
  };

  std::function<void(Worker&)> socket_thread;
  // control handshake (lock_2pl/caladan/server.cc:107-146): open `nports` fresh sockets, serve them, tell the client
  auto handle_control = [&](Worker& x, int fd, const sockaddr_in& who, int nports) {
    if (nports < 1 || nports > 1024) return;
    std::vector<int> fds;
    std::vector<uint8_t> resp(sizeof(int) + sizeof(uint16_t) * (size_t)nports);
    memcpy(resp.data(), &nports, sizeof(int));
    sockaddr_in any = srv;
    any.sin_port = 0;
    for (int i = 0; i < nports; i++) {
      int dfd = open_socket(any, false);
      if (dfd < 0) { for (int q : fds) close(q); return; }
      sockaddr_in got{};
      socklen_t gl = sizeof got;
      getsockname(dfd, (sockaddr*)&got, &gl);
      const uint16_t p = ntohs(got.sin_port);          // rt::UdpConn::LocalAddr().port is host order
      memcpy(resp.data() + sizeof(int) + sizeof(uint16_t) * (size_t)i, &p, sizeof p);
      fds.push_back(dfd);
    }
    {
      std::lock_guard<std::mutex> lk(mu);
      w.push_back(make_worker(std::move(fds), x.group, false));
      Worker* nw = w.back().get();
      nw->th = std::thread(socket_thread, std::ref(*nw));
    }
    sendto(fd, resp.data(), resp.size(), 0, (const sockaddr*)&who, sizeof who);
    x.controls++;
  };

  socket_thread = [&](Worker& x) {
    std::vector<pollfd> pfd(x.fds.size());
    while (!g_stop.load()) {
      // ---- receive (replaces net_recv): wait for the first datagram, then drain what has queued up ----
      for (int i = 0; i < x.dirty; i++) { x.hdr[i].msg_hdr.msg_namelen = sizeof(sockaddr_in); x.hdr[i].msg_len = 0; }   // what the last batch touched
      x.dirty = 0;
      for (size_t i = 0; i < x.fds.size(); i++) pfd[i] = {x.fds[i], POLLIN, 0};
      if (poll(pfd.data(), (nfds_t)pfd.size(), 200) <= 0) continue;     // timeout: look at the stop flag again
      int n = 0;
      const auto t0 = std::chrono::steady_clock::now();
      for (;;) {
        bool any = false;
        for (size_t i = 0; i < x.fds.size() && (unsigned)n < batch_max; i++) {
          const int m = recvmmsg(x.fds[i], x.hdr.data() + n, batch_max - (unsigned)n, MSG_DONTWAIT, nullptr);
          if (m > 0) { for (int q = 0; q < m; q++) x.from[n + q] = (int)i; n += m; any = true; }
        }
        if ((unsigned)n >= batch_max) break;
        if (!any && std::chrono::steady_clock::now() - t0 > std::chrono::microseconds(linger_us)) break;   // a short linger so that load builds batches
      }
      x.dirty = n;
      int keep = 0;                                   // a datagram of the wrong size cannot be a request of this server
      for (int i = 0; i < n; i++) {
        if (x.hdr[i].msg_len != msg) {
          int nports = 0;
          if (x.control && x.hdr[i].msg_len == sizeof(int)) {          // net_req{int nports}
            memcpy(&nports, x.buf.data() + (size_t)i * msg, sizeof(int));
            handle_control(x, x.fds[x.from[i]], x.peer[i], nports);
          } else x.dropped++;
          continue;
        }
        if (keep != i) {
          memcpy(x.buf.data() + (size_t)keep * msg, x.buf.data() + (size_t)i * msg, msg);
          x.peer[keep] = x.peer[i];
          x.from[keep] = x.from[i];
        }
        keep++;
      }
      if (keep == 0) continue;
      // ---- hand the batch to an engine thread and wait for the replies (they come back in x.buf) ----
      {
        std::unique_lock<std::mutex> lk(mu);
        x.n = keep;
        x.state = Worker::READY;
        cv_engine.notify_one();
        // (bounded waits: the signal handler only stores the flag, so a wakeup may be missed -- never a hang).  On a stop,
        // a batch no engine thread has taken is withdrawn, unserved; one that was taken is waited for and answered, so
        // that everything the state holds (and an --image-out saves) has been replied to.
        while (!cv_workers.wait_for(lk, std::chrono::milliseconds(100), [&] {
          return x.state == Worker::DONE || (g_stop.load() && x.state == Worker::READY);
        })) {}
        if (x.state != Worker::DONE) { x.state = Worker::FILLING; return; }
        x.state = Worker::FILLING;
      }
      // ---- send (replaces net_send): every reply goes back to the address, and from the socket, its request came to ----
      // (the headers still describe slot i <-> peer[i]; the kernel only touched msg_namelen / msg_len of the first n)
      for (int sent = 0; sent < keep;) {
        int run = 1;
        while (sent + run < keep && x.from[sent + run] == x.from[sent]) run++;
        for (int done = 0; done < run;) {
          const int r = sendmmsg(x.fds[x.from[sent]], x.hdr.data() + sent + done, (unsigned)(run - done), 0);
          if (r <= 0) { x.dropped += (uint64_t)(run - done); break; }
          done += r;
        }
        sent += run;
      }
      x.datagrams += (uint64_t)keep;
    }
  };

  // ---- sockets: as the reference sets them up, one per thread, all bound to the same port (one port per shard group) ----
  for (int g = 0; g < n_groups; g++) {
    sockaddr_in a = srv;
    a.sin_port = htons((uint16_t)(port + g));
    for (unsigned i = 0; i < n_sock; i++) {
      const int fd = open_socket(a, true);
      if (fd < 0) { perror("socket/bind"); return 1; }
      w.push_back(make_worker({fd}, g, true));
    }
  }
  signal(SIGINT, on_signal);
  signal(SIGTERM, on_signal);
  fprintf(stderr, "dint_udp_server: %s on %s:%d%s, %d GPU(s), %u sockets, batches of <= %u datagrams of %u bytes\n", argv[1],
          bind_addr.c_str(), port, n_groups > 1 ? " (+shard)" : "", gpus, n_sock * (unsigned)n_groups, batch_max, msg);
  {
    std::lock_guard<std::mutex> lk(mu);
    for (auto& x : w) x->th = std::thread(socket_thread, std::ref(*x));
  }

  // ---- utilisation channel (cpu_mon_func + cpu_mon_handler of the reference) ----
  std::atomic<double> ucores{0.0}, kcores{0.0};
  std::thread mon_sampler, mon_server;
  int mon_fd = -1;
  if (mon_port > 0) {
    sockaddr_in ma = srv;
    ma.sin_port = htons((uint16_t)mon_port);
    mon_fd = open_socket(ma, false);
    if (mon_fd < 0) { perror("mon socket/bind"); return 1; }
    timeval tv{0, 200000};
    setsockopt(mon_fd, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof tv);
    mon_sampler = std::thread([&] {
      rusage last{};
      getrusage(RUSAGE_SELF, &last);
      auto t_last = std::chrono::steady_clock::now();
      while (!g_stop.load()) {
        for (int i = 0; i < 10 && !g_stop.load(); i++) std::this_thread::sleep_for(std::chrono::milliseconds(100));
        rusage cur{};
        getrusage(RUSAGE_SELF, &cur);
        const auto t_now = std::chrono::steady_clock::now();
        const double dt = std::chrono::duration<double>(t_now - t_last).count();
        auto secs = [](const timeval& a, const timeval& b) { return (double)(a.tv_sec - b.tv_sec) + 1e-6 * (double)(a.tv_usec - b.tv_usec); };
        ucores.store(secs(cur.ru_utime, last.ru_utime) / dt);
        kcores.store(secs(cur.ru_stime, last.ru_stime) / dt);
        last = cur;
        t_last = t_now;
      }
    });
    mon_server = std::thread([&] {
      struct { double ucores, kcores; } m;
      while (!g_stop.load()) {
        sockaddr_in who{};
        socklen_t wl = sizeof who;
        if (recvfrom(mon_fd, &m, sizeof m, 0, (sockaddr*)&who, &wl) < 0) continue;      // timeout: look at the stop flag
        m.ucores = ucores.load();
        m.kcores = kcores.load();
        sendto(mon_fd, &m, sizeof m, 0, (const sockaddr*)&who, sizeof who);
      }
    });
  }

  // ---- engine threads: gather the ready batches, one submit, scatter the replies; two of them take turns ----
  std::mutex submit_mu;                               // the engine has ONE submitter at a time (include/dint_b200.h)
  auto engine_thread = [&]() {
    size_t arr_cap = (size_t)batch_max * 8;           // the array one submit sees: every ready batch, back to back (pinned)
    uint8_t* req = (uint8_t*)dint_host_alloc(arr_cap * msg);
    uint8_t* resp = (uint8_t*)dint_host_alloc(arr_cap * msg);
    std::vector<uint8_t> dst(arr_cap);
    std::vector<Worker*> taken;
    if (!req || !resp) { fprintf(stderr, "pinned allocation failed\n"); g_stop.store(true); return; }
    while (!g_stop.load()) {
      taken.clear();
      size_t n = 0;
      {
        std::unique_lock<std::mutex> lk(mu);
        cv_engine.wait_for(lk, std::chrono::milliseconds(200), [&] {
          for (const auto& x : w)
            if (x->state == Worker::READY) return true;
          return g_stop.load();
        });
        for (auto& x : w)                             // socket order: deterministic for a given set of ready batches
          if (x->state == Worker::READY && n + (size_t)x->n <= arr_cap) { x->state = Worker::IN_FLIGHT; taken.push_back(x.get()); n += (size_t)x->n; }
      }
      if (taken.empty()) continue;
      n = 0;
      for (Worker* x : taken) {                       // the batches back to back: ONE array for the engine
        memcpy(req + n * msg, x->buf.data(), (size_t)x->n * msg);
        memset(dst.data() + n, x->group, (size_t)x->n);
        n += (size_t)x->n;
      }
      int rc;
      {
        // replaces the switch(type) of the reference's server_loop for every gathered datagram, in array order
        std::lock_guard<std::mutex> sl(submit_mu);
        rc = cluster ? dint_cluster_submit(cluster, req, (uint64_t)n, by_dst ? dst.data() : nullptr, resp) : dint_submit(eng, req, (uint64_t)n, resp);
      }
      if (rc != DINT_OK && rc != DINT_EPROTO) {       // DINT_EPROTO: malformed records were answered with type 0xFF
        fprintf(stderr, "dint_udp_server: submit failed: %s\n", dint_last_error());
        g_stop.store(true);
      }
      if (rc == DINT_EPROTO) bad_batches++;
      submits++;
      size_t off = 0;
      for (Worker* x : taken) {
        memcpy(x->buf.data(), resp + off * msg, (size_t)x->n * msg);
        off += (size_t)x->n;
      }
      {
        std::lock_guard<std::mutex> lk(mu);
        for (Worker* x : taken) x->state = Worker::DONE;
      }
      cv_workers.notify_all();
    }
    dint_host_free(req);
    dint_host_free(resp);
  };
  std::thread second(engine_thread);
  engine_thread();
  second.join();
  {
    std::lock_guard<std::mutex> lk(mu);               // under the mutex: no worker sits between its predicate and its wait
    g_stop.store(true);
  }
  cv_workers.notify_all();
  uint64_t total = 0, dropped = 0, controls = 0;
  for (size_t i = 0;; i++) {                          // (control requests may still have been adding workers)
    Worker* x;
    {
      std::lock_guard<std::mutex> lk(mu);
      if (i >= w.size()) break;
      x = w[i].get();
    }
    if (x->th.joinable()) x->th.join();
    total += x->datagrams; dropped += x->dropped; controls += x->controls;
    for (int fd : x->fds) close(fd);
  }
  fprintf(stderr, "dint_udp_server: %llu datagrams in %llu submits (%.1f per submit), %llu dropped, %llu control requests, %llu submits with malformed records\n",
          (unsigned long long)total, (unsigned long long)submits.load(), submits.load() ? (double)total / (double)submits.load() : 0.0,
          (unsigned long long)dropped, (unsigned long long)controls, (unsigned long long)bad_batches.load());
  if (mon_sampler.joinable()) mon_sampler.join();
  if (mon_server.joinable()) mon_server.join();
  if (mon_fd >= 0) close(mon_fd);
  int exit_code = 0;
  if (!image_out.empty()) {                           // every engine thread has stopped and every reply was sent
    const int rc = cluster ? dint_cluster_image_save(cluster, image_out.c_str()) : dint_image_save(eng, image_out.c_str());
    if (rc != DINT_OK) { fprintf(stderr, "dint_udp_server: writing the image failed: %s\n", dint_last_error()); exit_code = 1; }
    else fprintf(stderr, "dint_udp_server: state image written to %s\n", image_out.c_str());
  }
  if (cluster) dint_cluster_destroy(cluster);
  if (eng) dint_destroy(eng);
  return exit_code;
}
