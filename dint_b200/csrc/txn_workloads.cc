// txn_workloads.cc -- (part of libdint_wl.so) the reference's TATP and SmallBank closed-loop clients as round-based
// generators on host cores.  The state machines themselves are txn_clients.cuh, shared with the clients that run on
// the GPU (dint_txn_clients_*); this file owns the client arrays, the counters and the C interface.
//
// dint_txn_next() emits a round -- each client's records contiguous, in the order the reference pushes them per
// shard -- plus the destination shard of every record; dint_txn_feed() hands the replies back in the same layout and
// advances every client's state machine.  dint_txn_set_draining() lets the clients finish the transactions they are in
// and start no new ones; an empty round is the end of such a drain, after which dint_txn_set_shards() may move them
// to another shard count.
#include <cstdint>
#include <cstring>
#include <vector>

#include "txn_clients.cuh"

using namespace txn;

struct dint_txn {
  int kind;                 // 4 = tatp, 5 = smallbank
  uint32_t n_clients;
  Cfg w;
  std::vector<TatpClient> tc;
  std::vector<SbClient> sc;
  uint64_t st_requests = 0, st_txns = 0, st_committed = 0, st_rounds = 0;
  uint64_t st_by_type[8] = {0}, st_commit_by_type[8] = {0};
  uint64_t st_lock[3] = {0};   // lock replies absorbed, of them kRejectLock, kRejectLockSameKey (client_lock.cc's lock_cnt,
                               // reject_sharing_cnt, reject_same_key_cnt)

  void begin(uint8_t type) { st_txns++; st_by_type[type]++; }          // the Sink of the shared state machines
  void commit(uint8_t type) { st_committed++; st_commit_by_type[type]++; }
  void lock_reply(uint8_t type) { st_lock[0]++; st_lock[1] += type == T_REJECT_LOCK; st_lock[2] += type == T_REJECT_LOCK_SAME_KEY; }
};

extern "C" {

// kind 4 (tatp): n_clients logical clients with gids [gid0, gid0 + n_clients); G shards; `subscribers`
// = kSubscriberNum of the key generator (reference 7,000,000; must equal the servers' population).
// kind 5 (smallbank): `subscribers` = kAccountNum (reference 24,000,000), hot set = 4 % of it (960,000).
dint_txn* dint_txn_create(int kind, uint32_t n_clients, uint32_t gid0, uint32_t n_shards, uint32_t subscribers) {
  // primary + 2 distinct backups need >= 3 shards; 1 = everything on one server (three copies of each write)
  if ((kind != 4 && kind != 5) || n_clients == 0 || n_shards == 0 || n_shards == 2 || n_shards > 8 || subscribers < 3) return nullptr;
  dint_txn* w = new dint_txn();
  w->kind = kind; w->n_clients = n_clients;
  w->w.G = n_shards; w->w.keys = subscribers; w->w.hot = 0;
  if (kind == 4) {
    w->tc.resize(n_clients);
    for (uint32_t i = 0; i < n_clients; i++) {
      w->tc[i].seed = (uint64_t)kSeedBase + gid0 + i;        // client_udp_shard.cc:1121
      tatp_begin(w->w, w->tc[i], *w);
    }
  } else {
    w->w.hot = (uint32_t)((uint64_t)subscribers * 960000 / 24000000);   // kHotAccountNum / kAccountNum
    if (w->w.hot < 2) w->w.hot = 2;
    w->sc.resize(n_clients);
    for (uint32_t i = 0; i < n_clients; i++) { w->sc[i].seed = (uint64_t)kSeedBase + gid0 + i; sb_begin(w->w, w->sc[i], *w); }
  }
  return w;
}
void dint_txn_destroy(dint_txn* w) { delete w; }
uint32_t dint_txn_max_round(const dint_txn* w) { return w->n_clients * kMaxRecords; }

// emits one round; returns the number of wire records.  req: capacity dint_txn_max_round() records;
// dst[i] = destination shard of record i.  An empty round (the end of a drain) is not counted.
uint64_t dint_txn_next(dint_txn* w, void* req, uint8_t* dst) {
  Out o{(uint8_t*)req, dst, 0, 0, w->kind == 4 ? (uint32_t)TM : (uint32_t)SMSZ};
  if (w->kind == 4) for (auto& c : w->tc) tatp_emit(w->w, c, o, *w);
  else for (auto& c : w->sc) sb_emit(w->w, c, o, *w);
  w->st_requests += o.n;
  if (o.n) w->st_rounds++;
  return o.n;
}
// on != 0: a client that finishes its transaction goes idle; 0: idle clients begin again at the next dint_txn_next
void dint_txn_set_draining(dint_txn* w, int on) { w->w.drain = on ? 1u : 0u; }
// the clients mid-transaction (not idle)
uint32_t dint_txn_busy(const dint_txn* w) {
  uint32_t n = 0;
  if (w->kind == 4) for (const auto& c : w->tc) n += c.txn != kIdle;
  else for (const auto& c : w->sc) n += c.txn != kIdle;
  return n;
}
// address every later record with key % G: only between transactions (busy == 0), G = 1 or 3..8.  0, or -22
// (EINVAL) with nothing changed.
int dint_txn_set_shards(dint_txn* w, uint32_t G) {
  if (G == 0 || G == 2 || G > 8 || dint_txn_busy(w) != 0) return -22;
  w->w.G = G;
  return 0;
}
void dint_txn_feed(dint_txn* w, const void* resp) {
  const uint8_t* r = (const uint8_t*)resp;
  // absorb may start a new transaction and must not see its own n_out
  if (w->kind == 4)
    for (auto& c : w->tc) { const uint32_t n = c.n_out; tatp_absorb(w->w, c, r, *w); r += (size_t)n * TM; }
  else
    for (auto& c : w->sc) { const uint32_t n = c.n_out; sb_absorb(w->w, c, r, *w); r += (size_t)n * SMSZ; }
}
// out: requests, transactions started, committed, rounds, then started-by-type[7], committed-by-type[7]
void dint_txn_stats(const dint_txn* w, uint64_t out[18]) {
  out[0] = w->st_requests; out[1] = w->st_txns; out[2] = w->st_committed; out[3] = w->st_rounds;
  for (int i = 0; i < 7; i++) { out[4 + i] = w->st_by_type[i]; out[11 + i] = w->st_commit_by_type[i]; }
}
// out: kAcquireLock replies absorbed, of them refused through false sharing (kRejectLock) and by a holder of the same
// key (kRejectLockSameKey): the counters behind tatp/caladan/client_lock.cc:403-428.  smallbank: zeros.
void dint_txn_lock_stats(const dint_txn* w, uint64_t out[3]) {
  for (int i = 0; i < 3; i++) out[i] = w->st_lock[i];
}

}  // extern "C"
