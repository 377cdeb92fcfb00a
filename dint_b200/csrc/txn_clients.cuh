// txn_clients.cuh -- the TATP and SmallBank closed-loop client state machines, stated ONCE for the host drivers
// (txn_workloads.cc, g++, libdint_wl.so) and the clients that run on the GPU (clients.cu, nvcc, dint_txn_clients_*).
//
// The reference: tatp/caladan/client_udp_shard.cc:177-1184 (seven transaction types, mix 35/35/10/2/14/2/2,
// tatp/udp/tatp.h:57-63) and smallbank/caladan/client_udp_shard.cc:169-1300 (six types, mix 15/15/15/25/15/15,
// hot-account skew smallbank/udp/smallbank.h:16-18,24-46), restated as round-based generators.
//
// A ROUND = every logical client has the requests of its current protocol step outstanding (1-9 wire records: the
// reference fans a step out to the shards in parallel and joins).  *_emit() appends a client's records -- in the order
// the reference pushes them per shard -- and the destination shard of each; *_absorb() takes the replies to exactly
// those records and advances the state machine.  Each client draws from the LCG fastrand(seed = 0xdeadbeef + gid)
// (tatp/udp/tatp.h:32-42), so a client's transaction stream is the reference's for that gid.
//
// Sharding generalised from 3 to G shards (SURVEY.md section 8(e)): primary p = key % G, backups (p+1) % G and
// (p+2) % G, log records to those same three; G = 3 is exactly the reference.
//
// Statistics go to a Sink: begin(type) when a transaction starts, commit(type) when one commits, lock_reply(type) for
// every absorbed reply to a TATP kAcquireLock.  One step (an absorb, then an emit) finishes at most one transaction,
// starts at most one and sees at most two lock replies, which the device sink relies on.
//
// Draining (Cfg::drain): a client that finishes a transaction while the drain word is set counts the commit and goes
// IDLE (txn == kIdle) instead of starting the next one.  An idle client emits and absorbs nothing; once the drain word
// is clear again it begins its next transaction in the emit step, then emits that transaction's first records.  Every
// draw happens in *_begin, so a drain changes when a client's transactions run, never which.  A round in which no
// client emits a record is the end of a drain: nobody serves or counts it.
//
// Under nvcc the kernels of the on-GPU clients follow (one thread per client; see the comment above them).
#pragma once
#include <cstdint>
#include <cstring>

#ifdef __CUDACC__
#define TXN_HD __host__ __device__ inline
#else
#define TXN_HD inline
#endif

namespace txn {

TXN_HD uint32_t fastrand(uint64_t* seed) {
  *seed = *seed * 1103515245ULL + 12345ULL;
  return (uint32_t)(*seed >> 32);
}
TXN_HD void put64(uint8_t* p, uint64_t v) { memcpy(p, &v, 8); }
TXN_HD uint64_t get64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
TXN_HD uint32_t get32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
TXN_HD void put32(uint8_t* p, uint32_t v) { memcpy(p, &v, 4); }
// float add in round-to-nearest, never contracted or reassociated: the device must reproduce the host's sums bit for bit
TXN_HD float fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}

constexpr uint32_t kMaxRecords = 9;      // records one client emits in one round (SmallBank: 3 written rows x 3 holders)
constexpr uint32_t kSeedBase = 0xdeadbeefu;   // client_udp_shard.cc:1121: seed = 0xdeadbeef + gid
// txn of an idle client: never a transaction type (0 is X_GET_SUB / B_AMALGAMATE, and zero-filled storage is the initial
// state)
constexpr uint8_t kIdle = 0xFF;

// ================================================ TATP ==============================================
// wire: {ord@0, type@1, table@2, key@3, val@11[40], ver@51}  (tatp/udp/net.h:57-65)
constexpr int TM = 55;
// T_REJECT_LOCK_SAME_KEY: only servers that keep holder keys send it (tatp/ebpf/lock_kern.c:297-298, proto.h:52)
enum { T_READ = 0, T_LOCK = 1, T_ABORT = 2, T_GRANT_READ = 4, T_NOT_EXIST = 6, T_GRANT_LOCK = 7, T_REJECT_LOCK = 8,
       T_REJECT_LOCK_SAME_KEY = 28, T_COMMIT_PRIM = 12, T_COMMIT_BCK = 13, T_COMMIT_LOG = 14, T_INSERT_PRIM = 18, T_INSERT_BCK = 19,
       T_DELETE_PRIM = 22, T_DELETE_BCK = 23, T_DELETE_LOG = 24 };
enum { TB_SUB = 0, TB_SEC = 1, TB_ACC = 2, TB_SF = 3, TB_CF = 4 };
enum { X_GET_SUB = 0, X_GET_ACC, X_GET_DEST, X_UPD_SUB, X_UPD_LOC, X_INS_CF, X_DEL_CF };

struct TMsg { uint8_t b[TM]; };

// Client state.  Plain data: zero-filled storage (value-initialised vector, cudaMemset) is the initial state.
struct TatpClient {
  uint64_t seed;
  uint8_t txn, phase, n_out;
  uint32_t s_id, vlr;
  uint8_t sf_type, start_time, end_time, cf_to_fetch;
  TMsg a, b, c, d;          // saved replies; roles depend on the transaction (see comments in tatp_emit)
  bool lock_a, lock_b;
};

// ================================================ SmallBank =========================================
// wire: {ord@0, type@1, table@2, key@3, val@11[8] = {u32 magic; float bal}, ver@19}  (smallbank/udp/net.h:43-52)
constexpr int SMSZ = 23;
enum { S_ACQ_S = 0, S_ACQ_X = 1, S_REL_S = 2, S_REL_X = 3, S_COMMIT_PRIM = 4, S_COMMIT_BCK = 5, S_COMMIT_LOG = 6,
       S_GRANT_S = 7, S_REJECT_S = 8, S_GRANT_X = 9, S_REJECT_X = 10 };
enum { B_AMALGAMATE = 0, B_BALANCE, B_DEPOSIT, B_SEND, B_TRANSACT, B_WRITECHECK };
enum { SP_ACQ = 0, SP_REL_ABORT, SP_LOG, SP_BCK, SP_PRIM, SP_RELEASE };
struct SbRow { uint8_t table, excl, write, granted; uint64_t acct; TMsg m; };
struct SbClient {
  uint64_t seed;
  uint8_t txn, phase, n_rows, n_out, rel_idx;
  SbRow r[3];
};

// The workload parameters every client shares.
struct Cfg {
  uint32_t G;              // shards
  uint32_t keys;           // tatp: kSubscriberNum; smallbank: kAccountNum
  uint32_t hot;            // smallbank: kHotAccountNum
  uint32_t drain;          // != 0: a client that finishes a transaction goes idle instead of starting the next
};
TXN_HD uint32_t prim(const Cfg& w, uint64_t key) { return (uint32_t)(key % w.G); }

// One client's records of one round: records n0..n-1 are this client's.
struct Out {
  uint8_t* req; uint8_t* dst; uint32_t n, n0, msz;
  // msg->ord = j, the record's index inside its shard's list of this client and step (Out::push of the reference)
  TXN_HD void push(const TMsg& m, uint32_t shard, bool set_ord) {
    uint8_t* p = req + (size_t)n * msz;
    memcpy(p, m.b, msz);
    if (set_ord) {
      uint32_t j = 0;
      for (uint32_t i = n0; i < n; i++) j += dst[i] == (uint8_t)shard;
      p[0] = (uint8_t)j;
    }
    dst[n++] = (uint8_t)shard;
  }
};

// Replication fan-out of up to three records.  Per-shard arrival order follows the reference's push order:
// log: for shard { rec0, rec1 } (:490-499); backups: rec0,rec1 -> +1 then rec0,rec1 -> +2 (:523-531).
TXN_HD void emit_log(const Cfg& w, Out& o, const TMsg* recs, int n, uint8_t type) {
  for (uint32_t s = 0; s < w.G; s++)
    for (int k = 0; k < n; k++) {
      const uint32_t p = prim(w, get64(recs[k].b + 3));
      for (uint32_t off = 0; off < 3; off++)
        if ((p + off) % w.G == s) { TMsg t = recs[k]; t.b[1] = type; o.push(t, s, false); }
    }
}
TXN_HD void emit_bck(const Cfg& w, Out& o, const TMsg* recs, int n, uint8_t type) {
  for (uint32_t s = 0; s < w.G; s++)
    for (uint32_t off = 1; off <= 2; off++)
      for (int k = 0; k < n; k++)
        if ((prim(w, get64(recs[k].b + 3)) + off) % w.G == s) { TMsg t = recs[k]; t.b[1] = type; o.push(t, s, false); }
}
TXN_HD void emit_prim(const Cfg& w, Out& o, const TMsg* recs, int n, uint8_t type) {
  for (uint32_t s = 0; s < w.G; s++)
    for (int k = 0; k < n; k++)
      if (prim(w, get64(recs[k].b + 3)) == s) { TMsg t = recs[k]; t.b[1] = type; o.push(t, s, false); }
}

// ---- TATP -------------------------------------------------------------------------------------------
TXN_HD uint64_t sub_nbr_of(uint32_t s_id) {            // tatp/udp/tatp.h:17-25,132-144
  uint64_t r = 0;
  for (int g = 0; g < 3; g++) {
    uint32_t i = s_id % 1000;
    s_id /= 1000;
    r |= ((uint64_t)(((i / 100) % 10) << 8 | ((i / 10) % 10) << 4 | (i % 10))) << (12 * g);
  }
  return r;
}

// tatp/udp/tatp.h:40-43: ((fastrand % S) | (fastrand & 1048575)) % S.  C++ leaves the order of the two draws
// unspecified; the reference's g++ build takes the LEFT one first, and so does this.
TXN_HD uint32_t nurand(const Cfg& w, uint64_t* seed) {
  const uint32_t a = fastrand(seed) % w.keys;
  const uint32_t b = fastrand(seed) & 1048575u;
  return (a | b) % w.keys;
}

// transaction mix (client_udp_shard.cc:1144, tatp.h:57-63): 35 35 10 2 14 2 2 percent
TXN_HD uint8_t tatp_pick(uint32_t x) {
  x %= 100;
  return x < 35 ? X_GET_SUB : x < 70 ? X_GET_ACC : x < 80 ? X_GET_DEST : x < 82 ? X_UPD_SUB : x < 96 ? X_UPD_LOC
                                                                                          : x < 98 ? X_INS_CF : X_DEL_CF;
}

template <class Sink>
TXN_HD void tatp_begin(const Cfg& w, TatpClient& c, Sink& sink) {
  c.txn = tatp_pick(fastrand(&c.seed));
  c.phase = 0;
  c.lock_a = c.lock_b = false;
  sink.begin(c.txn);
  switch (c.txn) {                                     // transaction parameters, in the reference's draw order
    case X_GET_SUB: c.s_id = nurand(w, &c.seed); break;
    case X_GET_ACC: c.s_id = nurand(w, &c.seed); c.sf_type = (uint8_t)((fastrand(&c.seed) & 3) + 1); break;
    case X_GET_DEST:
    case X_INS_CF:
      c.s_id = nurand(w, &c.seed);
      c.sf_type = (uint8_t)((fastrand(&c.seed) % 4) + 1);
      c.start_time = (uint8_t)((fastrand(&c.seed) % 3) * 8);
      c.end_time = (uint8_t)(fastrand(&c.seed) % 24);
      c.cf_to_fetch = (uint8_t)(c.start_time / 8 + 1);
      break;
    case X_UPD_SUB: c.s_id = nurand(w, &c.seed); c.sf_type = (uint8_t)((fastrand(&c.seed) % 4) + 1); break;
    case X_UPD_LOC: c.s_id = nurand(w, &c.seed); c.vlr = fastrand(&c.seed); break;
    default:  // X_DEL_CF
      c.s_id = nurand(w, &c.seed);
      c.sf_type = (uint8_t)((fastrand(&c.seed) % 4) + 1);
      c.start_time = (uint8_t)((fastrand(&c.seed) % 3) * 8);
      break;
  }
}
template <class Sink>
TXN_HD void tatp_finish(const Cfg& w, TatpClient& c, bool committed, Sink& sink) {
  if (committed) sink.commit(c.txn);
  if (w.drain) c.txn = kIdle;
  else tatp_begin(w, c, sink);
}

TXN_HD uint64_t k_sub(const TatpClient& c) { return c.s_id; }
TXN_HD uint64_t k_sf(const TatpClient& c) { return (uint64_t)c.s_id | ((uint64_t)c.sf_type << 32); }
TXN_HD uint64_t k_cf(const TatpClient& c, uint32_t st) { return k_sf(c) | ((uint64_t)st << 40); }
TXN_HD void mk(TMsg& m, uint8_t type, uint8_t table, uint64_t key) {
  memset(m.b, 0, TM);
  m.b[1] = type; m.b[2] = table; put64(m.b + 3, key);
}

// one protocol step of one client; an idle client begins its next transaction first unless the clients drain
template <class Sink>
TXN_HD void tatp_emit(const Cfg& w, TatpClient& c, Out& o, Sink& sink) {
  const uint32_t n0 = o.n;
  o.n0 = n0;
  if (c.txn == kIdle) {
    if (w.drain) { c.n_out = 0; return; }
    tatp_begin(w, c, sink);
  }
  TMsg m;
  switch (c.txn) {
    case X_GET_SUB: mk(m, T_READ, TB_SUB, k_sub(c)); o.push(m, prim(w, k_sub(c)), false); break;                 // :177-199
    case X_GET_ACC: mk(m, T_READ, TB_ACC, k_sf(c)); o.push(m, prim(w, k_sf(c)), false); break;                   // :305-331 (ai_type in sf_type)
    case X_GET_DEST:                                                                                               // :202-302
      if (c.phase == 0) { mk(m, T_READ, TB_SF, k_sf(c)); o.push(m, prim(w, k_sf(c)), false); }
      else for (uint32_t i = 0; i < c.cf_to_fetch; i++) { mk(m, T_READ, TB_CF, k_cf(c, i * 8)); o.push(m, prim(w, k_cf(c, i * 8)), true); }
      break;
    case X_UPD_SUB:                                                                                                // :334-571
      switch (c.phase) {
        case 0:   // a = sub read, b = sub lock, c = specfac read, d = specfac lock
          mk(m, T_READ, TB_SUB, k_sub(c)); o.push(m, prim(w, k_sub(c)), true);
          mk(m, T_LOCK, TB_SUB, k_sub(c)); o.push(m, prim(w, k_sub(c)), true);
          mk(m, T_READ, TB_SF, k_sf(c)); o.push(m, prim(w, k_sf(c)), true);
          mk(m, T_LOCK, TB_SF, k_sf(c)); o.push(m, prim(w, k_sf(c)), true);
          break;
        case 1: { TMsg t = c.b; t.b[1] = T_ABORT; o.push(t, prim(w, k_sub(c)), false); break; }                 // release sub lock
        case 2: { TMsg t = c.d; t.b[1] = T_ABORT; o.push(t, prim(w, k_sf(c)), false); break; }                  // release specfac lock
        case 3:   // verify
          mk(m, T_READ, TB_SUB, k_sub(c)); o.push(m, prim(w, k_sub(c)), true);
          mk(m, T_READ, TB_SF, k_sf(c)); o.push(m, prim(w, k_sf(c)), true);
          break;
        case 4: { TMsg rr[2] = {c.a, c.c}; emit_log(w, o, rr, 2, T_COMMIT_LOG); break; }      // :487-518
        case 5: { TMsg rr[2] = {c.a, c.c}; emit_bck(w, o, rr, 2, T_COMMIT_BCK); break; }      // :520-548
        default: { TMsg rr[2] = {c.a, c.c}; emit_prim(w, o, rr, 2, T_COMMIT_PRIM); break; }   // :550-568
      }
      break;
    case X_UPD_LOC:                                                                                                // :574-728
      switch (c.phase) {
        case 0: mk(m, T_READ, TB_SEC, sub_nbr_of(c.s_id)); o.push(m, prim(w, sub_nbr_of(c.s_id)), false); break;
        case 1:   // a = sub read, b = sub lock
          mk(m, T_READ, TB_SUB, k_sub(c)); o.push(m, prim(w, k_sub(c)), true);
          mk(m, T_LOCK, TB_SUB, k_sub(c)); o.push(m, prim(w, k_sub(c)), true);
          break;
        case 2: mk(m, T_READ, TB_SUB, k_sub(c)); o.push(m, prim(w, k_sub(c)), false); break;                     // verify
        case 3: { TMsg t = c.b; t.b[1] = T_ABORT; o.push(t, prim(w, k_sub(c)), false); break; }
        case 4: emit_log(w, o, &c.a, 1, T_COMMIT_LOG); break;
        case 5: emit_bck(w, o, &c.a, 1, T_COMMIT_BCK); break;
        default: emit_prim(w, o, &c.a, 1, T_COMMIT_PRIM); break;
      }
      break;
    case X_INS_CF:                                                                                                 // :731-951
      switch (c.phase) {
        case 0: mk(m, T_READ, TB_SEC, sub_nbr_of(c.s_id)); o.push(m, prim(w, sub_nbr_of(c.s_id)), false); break;
        case 1: mk(m, T_READ, TB_SF, k_sf(c)); o.push(m, prim(w, k_sf(c)), false); break;                        // c = specfac read
        case 2:   // a = callfwd read, b = callfwd lock
          mk(m, T_READ, TB_CF, k_cf(c, c.start_time)); o.push(m, prim(w, k_cf(c, c.start_time)), true);
          mk(m, T_LOCK, TB_CF, k_cf(c, c.start_time)); o.push(m, prim(w, k_cf(c, c.start_time)), true);
          break;
        case 3: { TMsg t = c.b; t.b[1] = T_ABORT; o.push(t, prim(w, k_cf(c, c.start_time)), false); break; }
        case 4:   // verify specfac version + callfwd still absent
          mk(m, T_READ, TB_SF, k_sf(c)); o.push(m, prim(w, k_sf(c)), true);
          mk(m, T_READ, TB_CF, k_cf(c, c.start_time)); o.push(m, prim(w, k_cf(c, c.start_time)), true);
          break;
        case 5: emit_log(w, o, &c.a, 1, T_COMMIT_LOG); break;
        case 6: emit_bck(w, o, &c.a, 1, T_INSERT_BCK); break;
        default: emit_prim(w, o, &c.a, 1, T_INSERT_PRIM); break;
      }
      break;
    default:  // X_DEL_CF                                                                                          // :954-1117
      switch (c.phase) {
        case 0: mk(m, T_READ, TB_SEC, sub_nbr_of(c.s_id)); o.push(m, prim(w, sub_nbr_of(c.s_id)), false); break;
        case 1:   // a = callfwd read, b = callfwd lock
          mk(m, T_READ, TB_CF, k_cf(c, c.start_time)); o.push(m, prim(w, k_cf(c, c.start_time)), true);
          mk(m, T_LOCK, TB_CF, k_cf(c, c.start_time)); o.push(m, prim(w, k_cf(c, c.start_time)), true);
          break;
        case 2: { TMsg t = c.b; t.b[1] = T_ABORT; o.push(t, prim(w, k_cf(c, c.start_time)), false); break; }
        case 3: mk(m, T_READ, TB_CF, k_cf(c, c.start_time)); o.push(m, prim(w, k_cf(c, c.start_time)), false); break;   // verify
        case 4: emit_log(w, o, &c.a, 1, T_DELETE_LOG); break;
        case 5: emit_bck(w, o, &c.a, 1, T_DELETE_BCK); break;
        default: emit_prim(w, o, &c.a, 1, T_DELETE_PRIM); break;
      }
      break;
  }
  c.n_out = (uint8_t)(o.n - n0);
}

TXN_HD void tatp_load(TMsg& m, const uint8_t* r, int i) { memcpy(m.b, r + (size_t)i * TM, TM); }
TXN_HD uint8_t tatp_type(const uint8_t* r, int i) { return r[(size_t)i * TM + 1]; }
TXN_HD uint32_t tatp_ver(const TMsg& m) { return get32(m.b + 51); }
// A lock refused by a holder of the same key aborts the transaction exactly as one refused through false sharing does.
// (The reference's client_lock.cc:741-749 leaves kRejectLockSameKey out of its final reply types and re-sends the lock
// message as a kRead: SURVEY.md, appendix of quirks.  That is not reproduced.)
TXN_HD bool tatp_lock_refused(uint8_t type) { return type == T_REJECT_LOCK || type == T_REJECT_LOCK_SAME_KEY; }

// r: the replies to the client's records of the last tatp_emit, in the same order
template <class Sink>
TXN_HD void tatp_absorb(const Cfg& w, TatpClient& c, const uint8_t* r, Sink& sink) {
  if (c.txn == kIdle) return;
  switch (c.txn) {
    case X_GET_SUB: tatp_finish(w, c, true, sink); break;
    case X_GET_ACC: tatp_finish(w, c, tatp_type(r, 0) == T_GRANT_READ, sink); break;
    case X_GET_DEST:
      if (c.phase == 0) {
        if (tatp_type(r, 0) == T_NOT_EXIST || r[11] == 0) tatp_finish(w, c, false, sink);   // record absent or is_active == 0 (:231-237)
        else c.phase = 1;
      } else {
        bool ok = false;
        for (uint32_t i = 0; i < c.cf_to_fetch; i++)
          if (tatp_type(r, i) == T_GRANT_READ && i * 8 <= c.start_time && c.end_time < r[(size_t)i * TM + 11]) ok = true;   // :287-297
        tatp_finish(w, c, ok, sink);
      }
      break;
    case X_UPD_SUB:
      switch (c.phase) {
        case 0:
          tatp_load(c.a, r, 0); tatp_load(c.b, r, 1); tatp_load(c.c, r, 2); tatp_load(c.d, r, 3);
          c.lock_a = tatp_type(r, 1) == T_GRANT_LOCK; c.lock_b = tatp_type(r, 3) == T_GRANT_LOCK;
          sink.lock_reply(tatp_type(r, 1)); sink.lock_reply(tatp_type(r, 3));   // client_lock.cc:718 lock_cnt += 2
          if (tatp_type(r, 2) == T_NOT_EXIST || !c.lock_a || !c.lock_b) {      // :400-420
            if (c.lock_a) c.phase = 1; else if (c.lock_b) c.phase = 2; else tatp_finish(w, c, false, sink);
          } else {
            uint16_t bits = (uint16_t)fastrand(&c.seed);                  // sub_val->bits (:425)
            memcpy(c.a.b + 11 + 30, &bits, 2);
            c.c.b[11 + 2] = (uint8_t)fastrand(&c.seed);                   // specfac_val->data_a (:429)
            c.phase = 3;
          }
          break;
        case 1: if (c.lock_b) c.phase = 2; else tatp_finish(w, c, false, sink); break;
        case 2: tatp_finish(w, c, false, sink); break;
        case 3:
          if (tatp_ver(c.a) != get32(r + 51) || tatp_ver(c.c) != get32(r + TM + 51)) { c.phase = 1; }   // abort both (:470-484)
          else {
            put32(c.a.b + 51, tatp_ver(c.a) + 1); put32(c.c.b + 51, tatp_ver(c.c) + 1);               // :487-488
            c.phase = 4;
          }
          break;
        case 4: c.phase = 5; break;
        case 5: c.phase = 6; break;
        default: tatp_finish(w, c, true, sink); break;
      }
      break;
    case X_UPD_LOC:
      switch (c.phase) {
        case 0: c.phase = 1; break;
        case 1:
          tatp_load(c.a, r, 0); tatp_load(c.b, r, 1);
          sink.lock_reply(tatp_type(r, 1));
          if (tatp_lock_refused(tatp_type(r, 1))) tatp_finish(w, c, false, sink);   // :642
          else { memcpy(c.a.b + 11 + 36, &c.vlr, 4); c.phase = 2; }        // sub_val->vlr_location (:646)
          break;
        case 2:
          if (get32(r + 51) != tatp_ver(c.a)) c.phase = 3;                 // :661-667
          else { put32(c.a.b + 51, tatp_ver(c.a) + 1); c.phase = 4; }
          break;
        case 3: tatp_finish(w, c, false, sink); break;
        case 4: c.phase = 5; break;
        case 5: c.phase = 6; break;
        default: tatp_finish(w, c, true, sink); break;
      }
      break;
    case X_INS_CF:
      switch (c.phase) {
        case 0: c.phase = 1; break;
        case 1: tatp_load(c.c, r, 0); if (tatp_type(r, 0) == T_NOT_EXIST) tatp_finish(w, c, false, sink); else c.phase = 2; break;   // :781
        case 2:
          tatp_load(c.a, r, 0); tatp_load(c.b, r, 1);
          sink.lock_reply(tatp_type(r, 1));
          if (tatp_type(r, 0) == T_GRANT_READ || tatp_lock_refused(tatp_type(r, 1))) {   // :831-841: row exists or lock refused
            if (tatp_type(r, 1) == T_GRANT_LOCK) c.phase = 3; else tatp_finish(w, c, false, sink);
          } else {
            c.a.b[11 + 1] = 101;                                           // numberx[0] = magic (:846)
            c.a.b[11 + 0] = c.end_time;                                    // end_time (:847)
            c.phase = 4;
          }
          break;
        case 3: tatp_finish(w, c, false, sink); break;
        case 4:
          if (tatp_ver(c.c) != get32(r + 51) || tatp_type(r, 1) == T_GRANT_READ) c.phase = 3;   // :884-891
          else { put32(c.a.b + 51, 0); c.phase = 5; }                      // :894 ver = 0
          break;
        case 5: c.phase = 6; break;
        case 6: c.phase = 7; break;
        default: tatp_finish(w, c, true, sink); break;
      }
      break;
    default:  // X_DEL_CF
      switch (c.phase) {
        case 0: c.phase = 1; break;
        case 1:
          tatp_load(c.a, r, 0); tatp_load(c.b, r, 1);
          sink.lock_reply(tatp_type(r, 1));
          if (tatp_type(r, 0) == T_NOT_EXIST || tatp_lock_refused(tatp_type(r, 1))) {   // :1024-1033
            if (tatp_type(r, 1) == T_GRANT_LOCK) c.phase = 2; else tatp_finish(w, c, false, sink);
          } else c.phase = 3;
          break;
        case 2: tatp_finish(w, c, false, sink); break;
        case 3:
          if (tatp_type(r, 0) == T_NOT_EXIST || get32(r + 51) != tatp_ver(c.a)) c.phase = 2;   // :1053-1060
          else c.phase = 4;
          break;
        case 4: c.phase = 5; break;
        case 5: c.phase = 6; break;
        default: tatp_finish(w, c, true, sink); break;
      }
      break;
  }
}

// ---- SmallBank --------------------------------------------------------------------------------------
TXN_HD float get_bal(const TMsg& m) { float f; memcpy(&f, m.b + 11 + 4, 4); return f; }
TXN_HD void set_bal(TMsg& m, float f) { memcpy(m.b + 11 + 4, &f, 4); }

TXN_HD void sb_get_account(const Cfg& w, uint64_t* seed, uint64_t* a) {                 // smallbank/udp/smallbank.h:24-30
  if (fastrand(seed) % 100 < 90) *a = fastrand(seed) % w.hot; else *a = fastrand(seed) % w.keys;
}
TXN_HD void sb_get_two_accounts(const Cfg& w, uint64_t* seed, uint64_t* a0, uint64_t* a1) {   // smallbank.h:32-46
  const uint32_t n = (fastrand(seed) % 100 < 90) ? w.hot : w.keys;
  *a0 = fastrand(seed) % n;
  *a1 = fastrand(seed) % n;
  while (*a1 == *a0) *a1 = fastrand(seed) % n;
}
TXN_HD void sb_row(SbRow& r, uint8_t table, bool excl, bool write, uint64_t acct) {
  r.table = table; r.excl = excl; r.write = write; r.granted = 0; r.acct = acct;
}
// transaction mix: 15 15 15 25 15 15 percent
TXN_HD uint8_t sb_pick(uint32_t x) {
  x %= 100;
  return x < 15 ? B_AMALGAMATE : x < 30 ? B_BALANCE : x < 45 ? B_DEPOSIT : x < 70 ? B_SEND : x < 85 ? B_TRANSACT : B_WRITECHECK;
}

template <class Sink>
TXN_HD void sb_begin(const Cfg& w, SbClient& c, Sink& sink) {
  c.txn = sb_pick(fastrand(&c.seed));
  c.phase = SP_ACQ;
  sink.begin(c.txn);
  uint64_t a0, a1;
  switch (c.txn) {
    case B_AMALGAMATE:       // client_udp_shard.cc:169-438: sav(a0) X, chk(a0) X, chk(a1) X, all written
      sb_get_two_accounts(w, &c.seed, &a0, &a1);
      c.n_rows = 3; sb_row(c.r[0], 0, true, true, a0); sb_row(c.r[1], 1, true, true, a0); sb_row(c.r[2], 1, true, true, a1);
      break;
    case B_BALANCE:          // :441-578: sav(a) S, chk(a) S, read only
      sb_get_account(w, &c.seed, &a0);
      c.n_rows = 2; sb_row(c.r[0], 0, false, false, a0); sb_row(c.r[1], 1, false, false, a0);
      break;
    case B_DEPOSIT:          // :581-684: chk(a) X += 1.3
      sb_get_account(w, &c.seed, &a0);
      c.n_rows = 1; sb_row(c.r[0], 1, true, true, a0);
      break;
    case B_SEND:             // :687-932: chk(a0) X, chk(a1) X, move 5.0
      sb_get_two_accounts(w, &c.seed, &a0, &a1);
      c.n_rows = 2; sb_row(c.r[0], 1, true, true, a0); sb_row(c.r[1], 1, true, true, a1);
      break;
    case B_TRANSACT:         // :935-1038: sav(a) X += 20.20
      sb_get_account(w, &c.seed, &a0);
      c.n_rows = 1; sb_row(c.r[0], 0, true, true, a0);
      break;
    default:                 // B_WRITECHECK :1041-1239: sav(a) S, chk(a) X -= 5 (+1 penalty)
      sb_get_account(w, &c.seed, &a0);
      c.n_rows = 2; sb_row(c.r[0], 0, false, false, a0); sb_row(c.r[1], 1, true, true, a0);
      break;
  }
}
template <class Sink>
TXN_HD void sb_finish(const Cfg& w, SbClient& c, bool ok, Sink& sink) {
  if (ok) sink.commit(c.txn);
  if (w.drain) c.txn = kIdle;
  else sb_begin(w, c, sink);
}

template <class Sink>
TXN_HD void sb_emit(const Cfg& w, SbClient& c, Out& o, Sink& sink) {
  const uint32_t n0 = o.n;
  o.n0 = n0;
  if (c.txn == kIdle) {
    if (w.drain) { c.n_out = 0; return; }
    sb_begin(w, c, sink);
  }
  switch (c.phase) {
    case SP_ACQ:
      for (int i = 0; i < c.n_rows; i++) {
        TMsg m; memset(m.b, 0, sizeof m.b);
        m.b[1] = c.r[i].excl ? S_ACQ_X : S_ACQ_S; m.b[2] = c.r[i].table; put64(m.b + 3, c.r[i].acct);
        o.push(m, (uint32_t)(c.r[i].acct % w.G), c.n_rows > 1);
      }
      break;
    case SP_REL_ABORT: {
      TMsg m = c.r[c.rel_idx].m; m.b[1] = c.r[c.rel_idx].excl ? S_REL_X : S_REL_S;
      o.push(m, (uint32_t)(c.r[c.rel_idx].acct % w.G), false);
      break;
    }
    case SP_LOG:
    case SP_BCK:
    case SP_PRIM: {
      TMsg rr[3];
      int nw = 0;
      for (int i = 0; i < c.n_rows; i++) if (c.r[i].write) rr[nw++] = c.r[i].m;
      if (c.phase == SP_LOG) emit_log(w, o, rr, nw, S_COMMIT_LOG);
      else if (c.phase == SP_BCK) emit_bck(w, o, rr, nw, S_COMMIT_BCK);
      else emit_prim(w, o, rr, nw, S_COMMIT_PRIM);
      break;
    }
    default:
      for (int i = 0; i < c.n_rows; i++) {
        TMsg m = c.r[i].m; m.b[1] = c.r[i].excl ? S_REL_X : S_REL_S;
        o.push(m, (uint32_t)(c.r[i].acct % w.G), c.n_rows > 1);
      }
      break;
  }
  c.n_out = (uint8_t)(o.n - n0);
}
TXN_HD int sb_next_granted(const SbClient& c, int from) {
  for (int i = from; i < c.n_rows; i++) if (c.r[i].granted) return i;
  return -1;
}
template <class Sink>
TXN_HD void sb_absorb(const Cfg& w, SbClient& c, const uint8_t* r, Sink& sink) {
  if (c.txn == kIdle) return;
  switch (c.phase) {
    case SP_ACQ: {
      bool all = true;
      for (int i = 0; i < c.n_rows; i++) {
        memcpy(c.r[i].m.b, r + (size_t)i * SMSZ, SMSZ);
        const uint8_t t = c.r[i].m.b[1];
        c.r[i].granted = (t == S_GRANT_S || t == S_GRANT_X);
        all &= (bool)c.r[i].granted;
      }
      bool logic_abort = false;
      if (all) {
        TMsg& m0 = c.r[0].m;
        switch (c.txn) {
          case B_AMALGAMATE:
            set_bal(c.r[2].m, fadd(get_bal(c.r[2].m), fadd(get_bal(c.r[0].m), get_bal(c.r[1].m))));
            set_bal(c.r[0].m, 0.f); set_bal(c.r[1].m, 0.f);
            break;
          case B_DEPOSIT: set_bal(m0, fadd(get_bal(m0), 1.3f)); break;
          case B_SEND:
            if (get_bal(c.r[0].m) < 5.0f) logic_abort = true;
            else { set_bal(c.r[0].m, fadd(get_bal(c.r[0].m), -5.0f)); set_bal(c.r[1].m, fadd(get_bal(c.r[1].m), 5.0f)); }
            break;
          case B_TRANSACT: set_bal(m0, fadd(get_bal(m0), 20.20f)); break;
          case B_WRITECHECK:
            if (fadd(get_bal(c.r[0].m), get_bal(c.r[1].m)) < 5.0f) set_bal(c.r[1].m, fadd(get_bal(c.r[1].m), -6.0f));
            else set_bal(c.r[1].m, fadd(get_bal(c.r[1].m), -5.0f));
            break;
          default: break;
        }
      }
      if (!all || logic_abort) {
        int g = sb_next_granted(c, 0);
        if (g < 0) sb_finish(w, c, false, sink); else { c.rel_idx = (uint8_t)g; c.phase = SP_REL_ABORT; }
      } else if (c.txn == B_BALANCE) {
        c.phase = SP_RELEASE;
      } else {
        for (int i = 0; i < c.n_rows; i++) if (c.r[i].write) put32(c.r[i].m.b + 19, get32(c.r[i].m.b + 19) + 1);   // ver++
        c.phase = SP_LOG;
      }
      break;
    }
    case SP_REL_ABORT: {
      int g = sb_next_granted(c, c.rel_idx + 1);
      if (g < 0) sb_finish(w, c, false, sink); else c.rel_idx = (uint8_t)g;
      break;
    }
    case SP_LOG: c.phase = SP_BCK; break;
    case SP_BCK: c.phase = SP_PRIM; break;
    case SP_PRIM: c.phase = SP_RELEASE; break;
    default: sb_finish(w, c, true, sink); break;
  }
}

// ==================================== the clients on the GPU ========================================
// One round of the clients of one cluster rank, three kernels on the rank's stream:
//   k_txn_step     one thread per client: absorb the client's replies to the last round (at the offset the last
//                  compaction gave it), advance the state machine, write this round's records into the client's
//                  fixed staging slots (kMaxRecords), and count them per 256-client tile and per destination shard;
//   k_txn_scan     one CTA: exclusive scan of the tile counts, then publish the round's size and its per-shard
//                  counts to a pinned host block (the host sizes the exchange slabs from them) and reset the latter;
//   k_txn_compact  one CTA per tile: each client's offset = tile base + scan inside the tile; each warp copies its 32
//                  clients' records, one client after the other, into the contiguous round req[] / dst[].
#ifdef __CUDACC__
}  // namespace txn
#include "kernels.cuh"
namespace txn {

struct DevClients {
  uint32_t n;                 // clients of this rank
  uint64_t gid0;              // gid of its first client
  Cfg w;
  void* cl;                   // TatpClient[n] or SbClient[n]
  uint8_t* stg;               // [n][kMaxRecords] records of this round, per client
  uint8_t* stg_dst;           // [n][kMaxRecords] their destination shards
  uint32_t* cnt;              // [n] records of this round, per client
  uint32_t* off;              // [n] offset of the client's first record in the round (= of its first reply)
  uint32_t* tile_sum;         // [tiles] records per tile; k_txn_scan turns it into the tiles' base offsets
  uint32_t* owner_cnt;        // [8] records of this round per destination shard
  unsigned long long* stats;  // [0, 7) transactions started per type, [7, 14) committed per type, [14, 17) lock replies
                              // absorbed, of them kRejectLock, kRejectLockSameKey
  uint8_t* req;               // the round, contiguous in client order
  uint8_t* dst;
  uint32_t* pub;              // mapped pinned host block: [0] records of the round, [1 + o] of them for shard o
};

constexpr uint32_t kDevStats = 17;   // words of DevClients::stats

// one step starts at most one transaction, commits at most one and sees at most two lock replies
struct DevSink {
  int began, done;
  uint32_t lock[3];             // lock replies, of them kRejectLock, kRejectLockSameKey
  __host__ __device__ void begin(uint8_t t) { began = t; }
  __host__ __device__ void commit(uint8_t t) { done = t; }
  __host__ __device__ void lock_reply(uint8_t t) { lock[0]++; lock[1] += t == T_REJECT_LOCK; lock[2] += t == T_REJECT_LOCK_SAME_KEY; }
};

template <int KIND>           // DINT_TATP (4) or DINT_SMALLBANK (5)
__global__ void __launch_bounds__(dint::kThreads, 1) k_txn_step(const DevClients d, const uint8_t* resp, int first) {
  constexpr uint32_t MSG = KIND == 4 ? TM : SMSZ;
  __shared__ uint32_t s_stats[kDevStats], s_own[8], s_sum;
  if (threadIdx.x < kDevStats) s_stats[threadIdx.x] = 0;
  if (threadIdx.x < 8) s_own[threadIdx.x] = 0;
  if (threadIdx.x == 0) s_sum = 0;
  __syncthreads();
  const uint32_t id = blockIdx.x * dint::kThreads + threadIdx.x;
  if (id < d.n) {
    DevSink sink{-1, -1, {0, 0, 0}};
    Out o{d.stg + (size_t)id * kMaxRecords * MSG, d.stg_dst + (size_t)id * kMaxRecords, 0, 0, MSG};
    if constexpr (KIND == 4) {
      TatpClient& c = ((TatpClient*)d.cl)[id];
      if (first) { c.seed = (uint64_t)kSeedBase + d.gid0 + id; tatp_begin(d.w, c, sink); }
      else tatp_absorb(d.w, c, resp + (size_t)d.off[id] * MSG, sink);
      tatp_emit(d.w, c, o, sink);
    } else {
      SbClient& c = ((SbClient*)d.cl)[id];
      if (first) { c.seed = (uint64_t)kSeedBase + d.gid0 + id; sb_begin(d.w, c, sink); }
      else sb_absorb(d.w, c, resp + (size_t)d.off[id] * MSG, sink);
      sb_emit(d.w, c, o, sink);
    }
    d.cnt[id] = o.n;
    for (uint32_t i = 0; i < o.n; i++) atomicAdd(&s_own[o.dst[i]], 1u);
    atomicAdd(&s_sum, o.n);
    if (sink.began >= 0) atomicAdd(&s_stats[sink.began], 1u);
    if (sink.done >= 0) atomicAdd(&s_stats[7 + sink.done], 1u);
    for (int i = 0; i < 3; i++) if (sink.lock[i]) atomicAdd(&s_stats[14 + i], sink.lock[i]);
  }
  __syncthreads();
  if (threadIdx.x < kDevStats && s_stats[threadIdx.x]) atomicAdd(&d.stats[threadIdx.x], (unsigned long long)s_stats[threadIdx.x]);
  if (threadIdx.x < 8 && s_own[threadIdx.x]) atomicAdd(&d.owner_cnt[threadIdx.x], s_own[threadIdx.x]);
  if (threadIdx.x == 0) d.tile_sum[blockIdx.x] = s_sum;
}

__global__ void __launch_bounds__(dint::kThreads) k_txn_scan(const DevClients d, uint32_t n_tiles) {
  __shared__ uint32_t wsum[dint::kThreads / 32];
  const uint32_t total = dint::cta_exclusive_scan<uint32_t>(d.tile_sum, d.tile_sum, n_tiles, 0u, wsum);
  if (threadIdx.x == 0) d.pub[0] = total;
  if (threadIdx.x < 8) {
    d.pub[1 + threadIdx.x] = d.owner_cnt[threadIdx.x];
    d.owner_cnt[threadIdx.x] = 0;
  }
}

template <uint32_t MSG>
__global__ void __launch_bounds__(dint::kThreads) k_txn_compact(const DevClients d) {
  __shared__ uint32_t wsum[dint::kThreads / 32];
  const uint32_t base = blockIdx.x * dint::kThreads;
  const uint32_t m = d.n - base < (uint32_t)dint::kThreads ? d.n - base : (uint32_t)dint::kThreads;
  (void)dint::cta_exclusive_scan<uint32_t>(d.cnt + base, d.off + base, m, d.tile_sum[blockIdx.x], wsum);
  const uint32_t id = base + threadIdx.x;
  const uint32_t my_k = id < d.n ? d.cnt[id] : 0, my_o = id < d.n ? d.off[id] : 0;
  const uint32_t lane = threadIdx.x & 31, w0 = id - lane;
  for (uint32_t j = 0; j < 32; j++) {
    const uint32_t k = __shfl_sync(0xffffffffu, my_k, j), o = __shfl_sync(0xffffffffu, my_o, j);
    if (!k) continue;
    const uint8_t* src = d.stg + (size_t)(w0 + j) * kMaxRecords * MSG;
    uint8_t* to = d.req + (size_t)o * MSG;
    for (uint32_t b = lane; b < k * MSG; b += 32) to[b] = src[b];
    if (lane < k) d.dst[o + lane] = d.stg_dst[(size_t)(w0 + j) * kMaxRecords + lane];
  }
}
#endif  // __CUDACC__

}  // namespace txn
