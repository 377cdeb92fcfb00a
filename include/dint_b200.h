/*
 * dint_b200.h -- C ABI of libdint_b200.so, the GPU-resident (H100) replacement for the per-request
 * server hot path of DINT (NSDI'24).
 *
 * The reference has no plugin/FFI API: the public interface of its hot path is the WIRE PROTOCOL
 * (one packed struct per UDP datagram; the reply is the same buffer with type/val/ver rewritten and
 * echoed to the sender) plus the server command line.  This ABI is what a transport front-end (UDP
 * recvmmsg/sendmmsg batcher, Caladan, DPDK burst loop) binds instead of calling the reference's
 * handler body one datagram at a time.  Each entry point cites the reference code it replaces
 * (paths relative to the DINT repository root).
 *
 * Semantics contract of dint_submit*: the n requests are processed AS IF one reference server
 * thread had received them one by one in index order (request i sees the effects of every j < i);
 * resp[i] is byte-for-byte the datagram that thread would have sent for req[i].  kRetry-class
 * replies, which exist only for thread-vs-thread spin contention in the reference
 * (lock_2pl/udp/server.cc:75-80, smallbank/udp/server_shard.cc:111-119), are never produced.
 *
 * There is no CPU fallback: every compute entry point fails with DINT_ENODEV when no CUDA device
 * is usable.
 */
#ifndef DINT_B200_H
#define DINT_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* Which reference server the engine stands in for. */
enum dint_kind {
  DINT_LOCK2PL = 0,   /* lock_2pl/udp/server.cc:55-123       wire: lock_2pl/udp/net.h:25-31   (6 B)  */
  DINT_FASST = 1,     /* lock_fasst/udp/server.cc:49-120     wire: lock_fasst/udp/net.h:25-31 (9 B)  */
  DINT_LOG = 2,       /* log_server/udp/server.cc:48-89      wire: log_server/udp/net.h:23-30 (53 B) */
  DINT_STORE = 3,     /* store/udp/server.cc:50-98           wire: store/udp/net.h:34-41      (53 B) */
  DINT_TATP = 4,      /* tatp/udp/server_shard.cc:88-211     wire: tatp/udp/net.h:57-65       (55 B) */
  DINT_SMALLBANK = 5, /* smallbank/udp/server_shard.cc:82-190 wire: smallbank/udp/net.h:43-52 (23 B) */
  DINT_NUM_KINDS = 6
};

/* Error codes (negative return values). */
enum {
  DINT_OK = 0,
  DINT_EINVAL = -22,  /* bad argument */
  DINT_ENOMEM = -12,  /* device/host allocation failed */
  DINT_ENODEV = -19,  /* no usable CUDA device (there is no CPU fallback) */
  DINT_EIO = -5,      /* a CUDA call failed; see dint_last_error() */
  DINT_EPROTO = -71   /* the batch held a request the reference would panic() on; the offending
                         replies carry type 0xFF, the rest of the batch was processed normally */
};

/*
 * Sizes the reference bakes in as constexpr (SURVEY.md section 5 "config / flags").  Defaults =
 * the reference constants; dint_default_cfg() fills them in.
 */
typedef struct dint_cfg {
  uint32_t lock_slots;     /* kLockHashSize 36,000,000: lock_2pl/udp/utils.h:16, lock_fasst/udp/utils.h:16 */
  uint32_t log_ring;       /* kMaxLogEntryNum 1,000,000: log_server/udp/utils.h:16, tatp/udp/kvs.h:19 */
  uint32_t subs_sizing;    /* kSubscriberNum that SIZES hash tables and lock-hash moduli:
                              store 2,000,000 (store/udp/tatp.h:10, server.cc:113),
                              tatp 7,000,000 (tatp/udp/tatp.h:28, server_shard.cc:75-79, tatp.h:12-14) */
  uint32_t subs_populate;  /* subscribers dint_populate() inserts (<= subs_sizing; a prefix of the
                              reference population, whose LCG streams are sequential in s_id) */
  uint32_t accts_sizing;   /* smallbank kAccountNum 24,000,000 (smallbank/udp/smallbank.h:17,
                              server_shard.cc:72-73, smallbank.h:10-14) */
  uint32_t accts_populate; /* accounts dint_populate() inserts */
  uint32_t n_shards;       /* key-space shards (GPUs); this engine owns lock slots / buckets with
                              slot % n_shards == shard_id.  1 = whole key space. */
  uint32_t shard_id;
  uint32_t chunk;          /* requests per internal launch group (0 = default 1<<20) */
  uint32_t kv_capacity_log2[5]; /* per-table open-addressing capacity (0 = auto: >= 2x expected keys) */
  uint32_t flags;          /* DINT_CFG_* option bits (below); the other bits are reserved */
  uint32_t txn_shards;     /* tatp / smallbank replica placement (tatp/caladan/client_udp_shard.cc:187,490-531 generalised
                              from 3 to G shards): 0 or 1 = this server holds every key (the reference: all three
                              shards populate everything); G > 3: dint_populate() keeps only keys whose primary
                              (key % G) is txn_shard_id, txn_shard_id-1 or txn_shard_id-2 (mod G) */
  uint32_t txn_shard_id;
  uint32_t reserved[2];
} dint_cfg;

/*
 * dint_cfg.flags bit 0, tatp only (dint_create / dint_cluster_create answer DINT_EINVAL for another kind): keep the
 * HOLDER'S KEY beside every lock bit, as the reference's eBPF lock server does (tatp/ebpf/lock_kern.c:12-16 `struct
 * txn_lock {u64 lock_bit; u64 key}`, written by a granted kAcquireLock, :292).  A refused kAcquireLock is then answered
 * kRejectLockSameKey (28) when the holder's key equals the request's -- a true conflict -- and kRejectLock (8) when it
 * differs -- false sharing: two keys hashed to one lock slot (lock_kern.c:289-298, tatp/ebpf/utils.h:73,
 * tatp/caladan/proto.h:52).  Releases leave the word alone, as the reference does (lock_kern.c:338,423,609,1119,1196);
 * it means something only while the bit is set.  Costs one u64 per lock slot (896 MB at the reference's sizes).
 * Without the bit nothing is allocated and every refused acquire is answered 8, as tatp/udp/server_shard.cc:123-132.
 */
#define DINT_CFG_LOCK_HOLDER_KEYS 1u

/*
 * dint_cfg.flags bits 1-2, store only (dint_create / dint_cluster_create answer DINT_EINVAL for another kind): answer as
 * the reference's eBPF store server does instead of its UDP server (store/udp/server.cc).  The eBPF server keeps a 4-slot
 * cache set per bucket in an XDP map (store/ebpf/store_kern.c:25-30, `struct cache_entry`, utils.h:58-66), answers hits
 * there, passes misses to a user-space `kvs` (store_user.c:127-165) and installs the table's answer from a TC egress
 * program (store_kern.c:302-373).  The tier leaks into the wire, so every reply depends on the hit / miss / eviction
 * history and the cache is modelled exactly:
 *   - a kSet that hits echoes the client's ver; one that misses returns the table's new version (store_user.c:148-149);
 *   - a kRead of an absent key whose bloom bit is clear is answered kNotExist with the request's ver (store_kern.c:88-94);
 *     a bloom false positive comes back kNotExist with ver = the eviction flag XDP put in ext_message.ver1 (:128-133);
 *   - a miss takes the first invalid slot, else the first clean one, else slot 0 (:116-125); a dirty victim is written
 *     back to the table first (kvs_set_evict, kvs.h:103-121), a clean one is overwritten;
 *   - kInsert fills a slot in XDP (dirty, the table does not see it) or, over a dirty victim, also writes back and
 *     inserts into the table (:226-297).  In the write-through variant (store_wt_kern.c:153-195) the cache keeps the
 *     CLIENT'S version of an inserted key while the table holds 0, a kSet invalidates the cached copy, and nothing is
 *     ever dirty.
 * kReject* replies (a set locked by another server thread) are never produced, as with kRetry elsewhere; a type other
 * than kRead / kSet / kInsert is answered 0xFF (DINT_EPROTO; store_user.c:164 panics).
 * The server starts EMPTY: dint_populate serves the eBPF client's kInsert stream (store/caladan/client_ebpf.cc:137-180,
 * 600 populate threads in thread order) through the tier, and dint_load serves its pairs as kInsert requests.
 * Costs 256 bytes of HBM per bucket (2.3 GB at the reference's 9,000,000 buckets).  Without these bits nothing is
 * allocated and the engine answers as store/udp/server.cc.
 * Limit: a key that reaches the table by kvs_insert twice (a second kInsert of a key the table already holds) is kept
 * twice by the reference's chained kvs (store/ebpf/kvs.h:75-101 never looks for an existing copy), which finds the copy
 * in its newest chain entry first; the engine's open-addressing table keeps both too but finds the first-inserted one.
 * Replies to such a key may then differ.  A key inserted once is served bit-exactly.  If the table is full (the
 * reference's chained table never is) the request that could not store its pair is answered 0xFF (DINT_EPROTO).
 */
#define DINT_CFG_STORE_EBPF_WB_BLOOM (1u << 1)  /* store/ebpf/store_kern.c: write-back cache + 64-bit bloom word per set */
#define DINT_CFG_STORE_EBPF_WB (2u << 1)        /* store/ebpf/store_wb_kern.c: write-back cache, no bloom word */
#define DINT_CFG_STORE_EBPF_WT (3u << 1)        /* store/ebpf/store_wt_kern.c + store_wt_user.c: write-through cache */
#define DINT_CFG_STORE_EBPF_MASK (3u << 1)
#define DINT_STORE_CACHE_ENTRY_BYTES 232         /* sizeof(struct cache_entry), store/ebpf/utils.h:58-66 */

/*
 * dint_cfg.flags bit 3, tatp only (dint_create / dint_cluster_create answer DINT_EINVAL for another kind, and
 * dint_create for n_shards > 1: place tatp shards with txn_shards): answer as the reference's eBPF TATP shard server
 * (tatp/ebpf/shard_kern.c with shard_user.c) instead of its UDP server (tatp/udp/server_shard.cc).  Together with
 * DINT_CFG_LOCK_HOLDER_KEYS it is tatp/ebpf/lock_kern.c.  The eBPF server keeps a 4-slot write-back cache set with a
 * bloom word per bucket of all five tables in XDP maps, answers hits and the lock traffic there, passes misses to a
 * user-space chained `kvs` and installs the answer from a TC egress program.  The tier leaks into the wire, so the
 * cache, the bloom words and the chained tables are modelled exactly:
 *   - sizes (tatp/ebpf/utils.h:11-21): subscriber and secondary subscriber S*3/2/4 buckets, access info, special
 *     facility AND call forwarding S*15/4/4 (the UDP server gives call forwarding S*45/8/4); 4 lock slots per bucket;
 *   - kRead: a hit answers from the set and sets the key's bloom bit (the top 6 bits of fasthash64(key)); a miss whose
 *     bit is clear is answered kNotExist with the request's ver; otherwise the table answers, after a dirty victim
 *     (first invalid slot, else first clean, else slot 0) was written back; a kNotExist from the table carries the
 *     eviction flag (0 / 1) in ver;
 *   - kCommitPrim / kCommitBck: a hit updates the set (ver + 1, dirty) and echoes the client's ver; a miss returns the
 *     TABLE's new version (0 when kvs_set inserted the row);
 *   - kInsertPrim / kInsertBck without a dirty victim put the row ONLY into the cache, dirty, with ver 0: the table
 *     sees it when it is evicted, by kvs_set(key, val, ver), which INCREMENTS the table's version when ver is 0 and
 *     inserts the row with version 0 when the table lacks it.  Over a dirty victim the row goes into the table too;
 *   - kDeletePrim / kDeleteBck: the first 8 value bytes of the reply are the bucket's rebuilt bloom word, one bit per
 *     CHAIN ENTRY of fasthash64 over its whole 32-byte key array (stale keys of invalid slots included,
 *     shard_user.c:94-104), so a later read of a key the table holds may be answered kNotExist;
 *   - a key inserted twice is kept twice by the chained table, and lookups find the copy nearer the chain's head;
 *   - the reference sends a kCommitBck miss back as its 108-byte ext_message (shard_kern.c:1231); the engine's reply
 *     is that datagram's first 55 bytes, which is what a client reading a struct message sees.
 * kReject* / kRetry replies (a set locked by another server thread) are never produced.  A type shard_user.c panics on
 * or a table >= 5 is answered 0xFF (DINT_EPROTO), as is a request that needed a chain entry when the engine's pool of
 * 1.5 entries per bucket was exhausted (counted in dint_tatp_cache_stats; the reference's calloc never fails); what
 * that request changed before the failed allocation (its cache set, a write-back) stays.
 * The server starts EMPTY: dint_populate serves the eBPF client's insert stream (tatp/caladan/client_ebpf_shard.cc:
 * 96-339, 600 populate threads in thread order) through the tier, kInsertPrim where this engine is the row's primary
 * (key % 3 == txn_shard_id; key % txn_shards when txn_shards > 3) and kInsertBck where it is a backup; dint_load serves
 * its pairs as kInsertBck requests (which leave the lock words alone).  Costs 256 bytes of HBM per bucket for the sets and 384 for the chain pool (6.4 + 9.6 GB at
 * S = 7,000,000).  Without the bit nothing is allocated and the engine answers as tatp/udp/server_shard.cc.
 * dint_lock_state / dint_lock_holder take the reference's lock slot (dint_lock_slot); dint_kv_get / dint_kv_count
 * answer from the chained tables, as kvs_get would.
 */
#define DINT_CFG_TATP_EBPF (1u << 3)
#define DINT_TATP_CHAIN_REC_BYTES 212   /* {u64 key[4]; u32 ver[4]; u8 valid[4]; u8 val[4][40]}, tatp/ebpf/kvs.h:13-19 */

/*
 * dint_cfg.flags bit 4, smallbank only (dint_create / dint_cluster_create answer DINT_EINVAL for another kind, and
 * dint_create for n_shards > 1: place smallbank shards with txn_shards): answer as the reference's eBPF SmallBank shard
 * server (smallbank/ebpf/shard_kern.c with shard_user.c) instead of its UDP server (smallbank/udp/server_shard.cc).
 * The eBPF server keeps the lock units {num_ex, num_sh} (the UDP server's 4H slots, lock_hash = h % 4H) and a 4-slot
 * write-back cache set per bucket of both tables (H = A*3/2/4 buckets) in XDP maps, answers the lock traffic and cache
 * hits there, passes misses to a user-space `kvs` and installs the answer from a TC egress program.  Per request:
 *   - kAcquireShared / kAcquireExclusive (0 / 1): a refusal (kRejectShared 8 / kRejectExclusive 10) changes nothing;
 *     the counters are SIGNED and refuse only when > 0 (num_ex > 0; num_ex > 0 or num_sh > 0), so a count a stray
 *     release took below zero refuses nothing (the UDP server's unsigned == 0 test refuses); a grant counts num_sh / num_ex BEFORE the cache is looked at; a hit answers kGrantShared 7
 *     / kGrantExclusive 9 with the set's val and ver; a miss picks a victim (first invalid slot, else first clean, else
 *     slot 0), writes a valid dirty victim back with kvs_set(key, val, ver) (which SETS the table's version to ver when
 *     ver != 0 and increments it when ver = 0), answers from the table and installs (key, val, ver) clean;
 *   - kReleaseShared / kReleaseExclusive (2 / 3): decrement, no floor, answer 11 / 12 (as the UDP server);
 *   - kCommitPrim / kCommitBck (4 / 5), no lock: a hit stores val, ver + 1, marks the slot dirty and ECHOES the client's
 *     ver (13 / 14); a miss writes a dirty victim back, then kvs_set(key, val, 0) increments the table's version, the
 *     reply carries the TABLE'S NEW VERSION and (key, val, new ver) is installed clean;
 *   - kCommitLog (6): appended to the 1,000,000-entry ring and answered 15 WHATEVER THE TABLE BYTE (the UDP server
 *     answers a table >= 2 with 0xFF);
 *   - kWarmupRead (17), never touching the lock units: a hit answers kGrantShared (7) with the set's val and ver, a miss
 *     goes through the table as above and answers kWarmupReadAck (18);
 *   - a table >= 2 on another type, or a type 7-16 or >= 18: answered 0xFF (DINT_EPROTO), no state change;
 *   - a KEY THE TABLE LACKS (an acquire, commit or warm-up miss): the reference's kvs_get / kvs_set panic and the server
 *     stops; the engine answers 0xFF, KEEPS what happened before the table lookup (the lock counter's increment, a dirty
 *     victim's write-back) and installs nothing.
 * Every reply is the 23-byte struct message; ord and the bytes the server does not write are echoed.  kRetry (16) and
 * the cache set's lock word serve contention between server threads and are never produced.
 * dint_populate inserts every account into the tables (shard_user.c:70-78, a prefix of accts_populate accounts), then
 * serves the eBPF client's warm-up stream (smallbank/caladan/client_ebpf_shard.cc:88-169: kWarmupRead of (saving, a)
 * then (checking, a) for every account a this shard replicates, ascending) through the tier, so the clients start on a
 * warm cache; dint_load inserts into the tables only and leaves the cache cold, as kvs_insert does.  dint_kv_get /
 * dint_kv_count answer from the tables, as kvs_get would (a dirty cached value is not visible there); dint_lock_state
 * takes the reference's lock slot (dint_lock_slot).  Costs 128 bytes of HBM per bucket (2.3 GB at A = 24,000,000).
 * Without the bit nothing is allocated and the engine answers as smallbank/udp/server_shard.cc.
 */
#define DINT_CFG_SMALLBANK_EBPF (1u << 4)
#define DINT_SMALLBANK_CACHE_ENTRY_BYTES 96   /* sizeof(struct cache_entry), smallbank/ebpf/utils.h:82-89 */

typedef struct dint_engine dint_engine;

/* Counters since create (or the last dint_reset_stats). */
typedef struct dint_stats {
  uint64_t requests;        /* requests processed */
  uint64_t chunks;          /* internal launch groups */
  uint64_t kernel_launches; /* kernels launched by this engine */
  uint64_t conflicted;      /* requests that took the ordered (intra-batch conflict) path */
  uint64_t max_run;         /* longest same-slot run seen on the ordered path */
  uint64_t errors;          /* requests answered with type 0xFF */
  uint64_t h2d_bytes, d2h_bytes;
  uint64_t kv_rebuilds;     /* KV tables rehashed to reclaim tombstones (the reference frees entries on delete:
                               store/udp/kvs.h:124-133) */
  /* which ordered-replay route the listed requests took (DESIGN.md section 3):
     ordered_fallbacks:  chunks whose listed requests overflowed a bucket and were replayed by the radix-sort fallback
     bucket_split_tasks: bucket-replay warp tasks that held more than a shared-memory slice and ran bucket by bucket
     writerless_chunks:  chunks without a single writer, whose conflict check was skipped altogether */
  uint64_t ordered_fallbacks;
  uint64_t bucket_split_tasks;
  uint64_t writerless_chunks;
} dint_stats;

/* Per-kernel device time, accumulated with CUDA events while profiling is on. */
typedef struct dint_kernel_time {
  char name[32];
  uint64_t launches;
  double total_ms;
} dint_kernel_time;

uint32_t dint_msg_size(int kind);                       /* sizeof(struct message) of that server */
void dint_default_cfg(int kind, dint_cfg *cfg);

/* Replaces server start-up: main() + net_init() + kvs_init()/array definitions
 * (lock_fasst/udp/server.cc:124-149, store/udp/server.cc:101-132, tatp/udp/server_shard.cc:71-85,278-320).
 * Allocates all state in HBM of CUDA device `device`; tables start EMPTY (see dint_populate). */
int dint_create(int kind, const dint_cfg *cfg, int device, dint_engine **out);
void dint_destroy(dint_engine *e);

/* Replaces populate_table / populate_*_table / populate_saving_and_checking_tables
 * (store/udp/tatp.h:45-66, tatp/udp/tatp.h:285-412, smallbank/udp/smallbank.h:105-127):
 * the same deterministic population, bytes the reference leaves uninitialised are zero. */
int dint_populate(dint_engine *e);

/* Bulk kvs_insert (store/udp/kvs.h:77-104) of n (key, value) pairs from HOST arrays into `table`;
 * vals is n * val_size bytes (40; smallbank 8).  Also the path that loads an image dumped from
 * another server.  Keys must not already exist (the reference's insert never checks either). */
int dint_load(dint_engine *e, int table, const uint64_t *keys, const void *vals, uint64_t n);

/* Replaces the `while (1) { net_recv; handler body; net_send; }` loop for a batch
 * (lock_2pl/udp/server.cc:70-122, lock_fasst/udp/server.cc:78-119, log_server/udp/server.cc:73-88,
 * store/udp/server.cc:75-97, tatp/udp/server_shard.cc:113-210, smallbank/udp/server_shard.cc:107-189).
 * req/resp: HOST arrays of n packed wire structs (resp may alias req).  Copies in, computes on the
 * GPU, copies out, returns when resp is complete.  Returns 0, DINT_EPROTO, or another error. */
int dint_submit(dint_engine *e, const void *req, uint64_t n, void *resp);

/* Same, with DEVICE arrays (16-byte aligned), asynchronous on `cuda_stream` (a cudaStream_t; NULL = the
 * legacy default stream, as everywhere in CUDA).  Successive calls must be issued on streams that
 * order them (the engine's state is one sequential history).  Request errors surface at the next
 * dint_sync()/dint_get_stats(). */
int dint_submit_device(dint_engine *e, const void *req_dev, uint64_t n, void *resp_dev, void *cuda_stream);
/* Multi-GPU routing helper (SURVEY.md section 8(e)): owner[i] = shard that owns request i's group
 * (lock slot / bucket: fasthash64 % size % n_shards -- the same modulus the single server would use, so
 * collision behaviour is unchanged by sharding); 0xFF for records no shard owns (invalid / log-only
 * requests are served by whoever receives them: owner = shard_id).  Device pointers, async on stream. */
int dint_route_owner(dint_engine *e, const void *req_dev, uint64_t n, uint8_t *owner_dev, void *cuda_stream);
/* Dispatch / combine for the multi-GPU exchange.  dint_route_partition: stable partition of n wire records by
 * owner_dev[i] (< n_shards; from dint_route_owner, or chosen by the client as in tatp / smallbank) into
 * sorted_dev (grouped by shard, each group in original order); perm_dev[pos] = original index;
 * counts_dev[0..n_shards) = records per shard.  dint_route_unpermute: out_dev[perm[pos]] = sorted_dev[pos].
 * All pointers are device pointers; asynchronous on cuda_stream. */
int dint_route_partition(dint_engine *e, const void *req_dev, const uint8_t *owner_dev, uint64_t n, uint32_t n_shards,
                         void *sorted_dev, uint32_t *perm_dev, uint32_t *counts_dev, void *cuda_stream);
/* Fixed-capacity dispatch / combine (no host round trip for the split sizes), local or over NVLink peer memory.
 * Every source rank sends every shard o one SLAB of `cap` records: its records for o first, in request order,
 * then padding records (every byte 0xFE: a padding record is answered unchanged and touches nothing).
 *   dint_route_dispatch: ONE kernel, one pass over the batch (single-pass prefix sums by decoupled look-back; n < 2^27).
 *     owner_in_dev = client-chosen shard per record (tatp / smallbank
 *     placement) or NULL = computed as dint_route_owner would (needs n_shards == cfg.n_shards).  slab_ptrs->p[o] =
 *     device address of THIS source's slab for shard o: inside a local send buffer (then exchange the slabs with
 *     an all-to-all) or inside rank o's receive buffer mapped over NVLink (then no collective is needed: with
 *     sig_ptrs != NULL the kernel's last CTA release-stores `epoch` to word `rank` of sig_ptrs->p[o] for every o).
 *     Outputs for the combine: owner_dev[n] (one byte per record, 0xFF = undeliverable) and tilebase_dev
 *     [ceil(n / dint_route_tile_records())][8].  flags_dev[0] += records that did not fit their slab.
 *   dint_route_combine: reply_slab_ptrs->p[o] = where shard o's replies to THIS source's slab are (local receive
 *     buffer or rank o's reply buffer over NVLink); out_dev[i] = reply to request i (0xFF bytes if undelivered).
 * The reference does this routing in its clients (e.g. `key % kNumServers` before sendto,
 * tatp/caladan/client_ebpf_shard.cc); with this call any rank may receive any request. */
typedef struct dint_peer_ptrs { uint64_t p[8]; } dint_peer_ptrs;
uint32_t dint_route_tile_records(dint_engine *e);
int dint_route_dispatch(dint_engine *e, const void *req_dev, const uint8_t *owner_in_dev, uint64_t n, uint32_t n_shards,
                        uint32_t rank, uint32_t cap, const dint_peer_ptrs *slab_ptrs, const dint_peer_ptrs *sig_ptrs,
                        uint32_t epoch, uint8_t *owner_dev, uint32_t *tilebase_dev, uint32_t *flags_dev, void *cuda_stream);
int dint_route_combine(dint_engine *e, const dint_peer_ptrs *reply_slab_ptrs, const uint8_t *owner_dev,
                       const uint32_t *tilebase_dev, uint64_t n, uint32_t n_shards, uint32_t cap, void *out_dev,
                       void *cuda_stream);
/* Epoch flags for the exchange over peer memory (one process per GPU; the buffers are each rank's
 * symmetric-memory regions mapped into this process; sig_ptrs->p[o] = rank o's signal words [n_shards] u32):
 *   dint_p2p_wait:    blocks the stream until local_sig[0..n_shards) have all reached epoch (acquire).
 *   dint_p2p_signal:  release-signals epoch to every peer's sig[rank] (e.g. replies ready in my reply buffer).
 * flags_dev[1] = 1 if a wait timed out. */
int dint_p2p_wait(dint_engine *e, const uint32_t *local_sig_dev, uint32_t n_shards, uint32_t epoch, uint32_t *flags_dev,
                  void *cuda_stream);
int dint_p2p_signal(dint_engine *e, const dint_peer_ptrs *sig_ptrs, uint32_t n_shards, uint32_t rank, uint32_t epoch,
                    void *cuda_stream);
/* The whole sharded step over NVLink peer memory, driven from ONE host call per sequence of batches (what
 * dint_b200/shard.py uses at N > 1, one process per GPU).  Every rank owns n_sets (2..4) buffer sets {inbox, return
 * buffer}, each n_shards * cap records (cap a multiple of 128), plus one 256-byte signal block (epoch words: requests
 * written [n_sets][8] at +0, replies written [8] at +128), all in memory its peers map (CUDA IPC / torch symmetric memory), zeroed once.
 *   inbox_sets[s].p[o], retbox_sets[s].p[o]: device address of rank o's set s; sig_blocks->p[o]: rank o's block.
 * dint_shard_submit_many: k batches of n (<= max_n) records each, the same k on every rank; batch j+1 is partitioned
 * into the OWNERS' inboxes (dint_route_dispatch) while batch j runs through the local engine on cuda_stream -- its
 * apply kernel stores every reply tile straight into the SOURCE's return buffer (posted stores) -- and the replies of
 * batch j-1 are put back in request order from the local return buffer (dint_route_combine); out_dev[j] is complete
 * when cuda_stream reaches the end of the call.  The engine sees the batches in order, so the result equals k
 * sequential collective steps.  dst_dev: NULL, or per batch the client-chosen shard of every record.
 * dint_shard_submit_host: the same with HOST buffers (pinned recommended): H2D | dispatch | engine | combine | D2H
 * pipelined n_sets deep; returns when every out_host[j] is complete.
 * dint_shard_flags (synchronises): [0] records that overflowed a slab, [1] timed-out waits, since the last call;
 * both must be 0 for the replies to stand. */
typedef struct dint_shard_ctx dint_shard_ctx;
int dint_shard_create(dint_engine *e, uint32_t n_shards, uint32_t rank, uint32_t cap, uint32_t n_sets,
                      const dint_peer_ptrs *inbox_sets, const dint_peer_ptrs *retbox_sets,
                      const dint_peer_ptrs *sig_blocks, uint64_t max_n, dint_shard_ctx **out);
void dint_shard_destroy(dint_shard_ctx *c);
int dint_shard_submit_many(dint_shard_ctx *c, uint32_t k, const void *const *req_dev, const uint8_t *const *dst_dev, uint64_t n,
                           void *const *out_dev, void *cuda_stream);
/* Batches of different sizes in one pipelined sequence (tatp / smallbank rounds): n[j] records in batch j (may differ
 * between ranks) and cap[j] = the slab capacity batch j uses (a multiple of 128, <= the cap of dint_shard_create, THE SAME
 * ON EVERY RANK; NULL or 0 = the full capacity): sized to the batch, the owners do not wade through padding. */
int dint_shard_submit_many_v(dint_shard_ctx *c, uint32_t k, const void *const *req_dev, const uint8_t *const *dst_dev,
                             const uint64_t *n, const uint32_t *cap, void *const *out_dev, void *cuda_stream);
int dint_shard_submit_host(dint_shard_ctx *c, uint32_t k, const void *const *req_host, const uint8_t *const *dst_host, uint64_t n,
                           void *const *out_host);
int dint_shard_flags(dint_shard_ctx *c, uint32_t out[2]);
/* Slab overflow (more records of one source for one owner than `cap`): the source flags it to EVERY owner with the
 * batch, and from that batch on no shard serves anything -- the state stays exactly what it was after the last complete
 * batch.  dint_shard_recover (call on every rank, synchronises): *first_unserved = index, inside the last submit call of
 * k_last batches, of the first batch left unserved (0xffffffff: none); clears the condition.  Serve the unserved
 * batches again in pieces of at most `cap` records per rank -- those cannot overflow.  (dint_cluster_submit does this.) */
int dint_shard_recover(dint_shard_ctx *c, uint32_t k_last, uint32_t *first_unserved);

/*
 * Multi-GPU server in ONE process: SURVEY.md section 8(b)'s `dint_create(kind, cfg, n_gpus)` / `dint_submit(e, req, n,
 * dst_shard, resp)`.  This is what a C/C++ transport front-end binds to serve one key space from all GPUs of a box
 * (the reference runs one `server_shard <id>` process per machine and lets the CLIENT pick the shard:
 * tatp/udp/server_shard.cc:278-320, tatp/caladan/client_udp_shard.cc:187,490-531).
 *   dint_cluster_create: n_gpus shard engines; devices[i] = CUDA ordinal of shard i (NULL: 0..n_gpus-1).  All
 *     ordinals distinct (peer access over NVLink is enabled between them), or all the same (several shards resident
 *     on one GPU: same results, used by the 1-GPU tests).  max_batch = records per shard and round (0 = 262144).
 *     lock_2pl / lock_fasst / store: shard i owns the lock slots / buckets with slot % n_gpus == i -- the slot ONE
 *     reference server would compute, so the cluster answers exactly like ONE server.  tatp / smallbank: shard i
 *     is `server_shard i+1` of an n_gpus-machine deployment (primary key % n_gpus, backups +1 and +2; n_gpus = 1 or
 *     >= 3) and holds only the keys it is a replica of.
 *   dint_cluster_submit: req/resp are HOST arrays of n wire structs; dst_shard[i] (tatp / smallbank: required, the
 *     shard the client would have sent record i to; other kinds: NULL) -- resp[i] answers req[i]; semantics: every
 *     shard sees its records in index order.  Keys skewed beyond the slack of the exchange slabs (all records of
 *     a round hashing to one shard) are handled: the round that does not fit is served again in smaller pieces.
 *     Returns 0, DINT_EPROTO, or an error; never blocks on the network.
 */
typedef struct dint_cluster dint_cluster;
int dint_cluster_create(int kind, const dint_cfg *cfg, int n_gpus, const int *devices, uint64_t max_batch, dint_cluster **out);
int dint_cluster_populate(dint_cluster *c);
int dint_cluster_submit(dint_cluster *c, const void *req, uint64_t n, const uint8_t *dst_shard, void *resp);
dint_engine *dint_cluster_engine(dint_cluster *c, int shard);   /* state inspection of one shard */
uint32_t dint_cluster_size(dint_cluster *c);
uint64_t dint_cluster_overflow_retries(dint_cluster *c);   /* submit calls that met a slab overflow (recovered, see dint_shard_recover) */
void dint_cluster_destroy(dint_cluster *c);
int dint_route_unpermute(dint_engine *e, const void *sorted_dev, const uint32_t *perm_dev, uint64_t n, void *out_dev,
                         void *cuda_stream);
int dint_sync(dint_engine *e);   /* waits for everything submitted on this engine's device */

/* ---- state inspection: parity of the final server state, not only of the wire ------------------ */
/* kvs_get on the device table (store/udp/kvs.h:37-55): 0 = found, 1 = not found. */
int dint_kv_get(dint_engine *e, int table, uint64_t key, void *val, uint32_t *ver);
/* Cache set `bucket` (fasthash64(key) % 9,000,000 at the reference's sizes) of a store engine with the eBPF cache tier,
 * written to `out` as the reference's struct cache_entry (232 bytes: key[4], val[4][40], ver[4], valid[4], dirty[4],
 * bloom_filter, lock = 0).  DINT_EINVAL without the tier or for a bucket another shard owns. */
int dint_store_cache_set(dint_engine *e, uint32_t bucket, void *out);
/* The tier's counters since create: out[0] requests answered from the cache (hits), [1] bloom negatives, [2] requests
 * served by the backing table (the user-space path), [3] dirty victims written back, [4] slots filled (installs and
 * cached inserts). */
int dint_store_cache_stats(dint_engine *e, uint64_t out[5]);
/* Cache set `bucket` (fasthash64(key) % the table's bucket count) of table `table` of a tatp engine with
 * DINT_CFG_TATP_EBPF, as the reference's struct cache_entry (232 bytes, tatp/ebpf/utils.h:103-111; lock = 0). */
int dint_tatp_cache_set(dint_engine *e, int table, uint32_t bucket, void *out);
/* The chain of that bucket, head first: *n = its length, and the first min(n, max) entries written to `out` as
 * DINT_TATP_CHAIN_REC_BYTES records (stale keys of invalid slots as the table left them). */
int dint_tatp_chain(dint_engine *e, int table, uint32_t bucket, void *out, uint32_t max, uint32_t *n);
/* The tier's counters since create: out[0] requests answered from the cache (hits), [1] bloom negatives, [2] requests
 * served by the user-space path, [3] dirty victims written back, [4] slots filled, [5] chain entries allocated from
 * the pool, [6] entries reused from the bucket's freed ones, [7] entries freed, [8] allocations that failed. */
int dint_tatp_cache_stats(dint_engine *e, uint64_t out[9]);
/* Cache set `bucket` (fasthash64(key) % A*3/2/4) of table `table` of a smallbank engine with DINT_CFG_SMALLBANK_EBPF,
 * as the reference's struct cache_entry (96 bytes; lock = 0). */
int dint_smallbank_cache_set(dint_engine *e, int table, uint32_t bucket, void *out);
/* The tier's counters since create: out[0] requests answered from the cache (hits), [1] requests served by the
 * user-space path (misses), [2] dirty victims written back, [3] slots installed.  Missing keys count in
 * dint_stats.errors. */
int dint_smallbank_cache_stats(dint_engine *e, uint64_t out[4]);
int64_t dint_kv_count(dint_engine *e, int table);
/* lock_2pl: out = {num_ex, num_sh}; lock_fasst: {lock, ver}; tatp: {lock, 0}; smallbank: {num_ex, num_sh} */
int dint_lock_state(dint_engine *e, int table, uint32_t slot, uint32_t out[2]);
/* tatp with DINT_CFG_LOCK_HOLDER_KEYS: the key the last granted kAcquireLock left in the slot (tatp/ebpf/lock_kern.c:292;
 * 0 = never granted; stale once dint_lock_state says the slot is free).  DINT_EINVAL without the option. */
int dint_lock_holder(dint_engine *e, int table, uint32_t slot, uint64_t *key);
/* slot the reference would compute for a lock id / key (fasthash64 % size) -- for tests */
uint32_t dint_lock_slot(dint_engine *e, int table, uint64_t key_or_lid);
/* copies ring 0 of the commit log (log_ring entries of dint_log_entry_size bytes, laid out as the
 * reference's struct log_entry) and the number of appends so far */
int dint_dump_log(dint_engine *e, void *out, uint64_t *appended);
uint32_t dint_log_entry_size(int kind);

/* Checkpoint / restore of the whole server state of one engine (lock words, versions, counters, KV tables, log ring),
 * device to device.  The reference has no such facility (its state dies with the process); a batched server can take
 * one between two calls at HBM copy speed.  dint_snapshot_restore is asynchronous on cuda_stream and must be ordered
 * between submit calls; it fails if a KV table was rehashed since the snapshot. */
typedef struct dint_snapshot dint_snapshot;
int dint_snapshot_create(dint_engine *e, dint_snapshot **out);
int dint_snapshot_restore(dint_snapshot *s, void *cuda_stream);
void dint_snapshot_destroy(dint_snapshot *s);

/*
 * State images: the same state as a snapshot (the regions dint_snapshot_create copies), saved to a FILE, packed and
 * checksummed on the device, and opened again as a new engine -- in another process, on another device, in a later
 * session.  The reference has no counterpart (its state dies with the process).
 *   dint_image_save: quiesces the engine as dint_snapshot_create does and writes `path`.  The file is written as
 *     path.tmp, fsynced, renamed, and the directory fsynced, so a crash never leaves a half image under the final name.
 *     It stages through three 64 MiB device buffers of the engine's host ring and three pinned host buffers, all
 *     released when the call returns.  Block b+1 is packed
 *     while block b is copied to pinned host memory and block b-1 is written.
 *   dint_image_open: checks the header before any CUDA call, creates an engine on `device` from the saved dint_cfg with
 *     every KV table at its saved capacity (the tombstone rehash may have doubled it since create), WITHOUT population or
 *     warm-up, and streams read | copy | check + unpack.  The engine answers every later request as the saved one would.
 *     Any failure returns no engine (*out = NULL):
 *       DINT_EINVAL  bad magic or format version, unknown kind or option flag, a region size this build would lay
 *                    out differently, or bytes after the last block;
 *       DINT_EIO     a file that cannot be opened, a short read, an I/O error, or a checksum mismatch.
 *     dint_last_error() names the file and, for a block, its region and block index.
 *   dint_cluster_image_save: directory `dir` (created if missing) holds shard-<r>.img of every shard and, written last,
 *     `manifest` {magic "DINTCLU1", u32 version, kind, shards, 0, the dint_cfg the cluster was created from, u32 0}.
 *     An earlier manifest in `dir` is removed (and the removal made durable) before the first shard image is replaced,
 *     so a save that stops part-way leaves a directory that dint_cluster_image_open refuses, never one whose shards
 *     were saved at different moments.
 *   dint_cluster_image_open: n_gpus must equal the manifest's shard count, and every shard file must exist; devices and
 *     max_batch as dint_cluster_create (all ordinals distinct, or all the same).
 *   A one-process-per-GPU deployment (dint_b200/shard.py) saves and opens each rank's engine with dint_image_save /
 *     dint_image_open and then calls dint_shard_create as usual.
 *   dint_image_times: the last image call of this thread, in seconds: [0] wall, [1] pack / unpack kernels (CUDA events),
 *     [2] device <-> host copies (CUDA events), [3] file reads and writes (host clock).
 * Not part of an image: dint_stats and the cache tiers' statistics (counters), client state (dint_clients,
 * dint_txn_clients, dint_cluster_clients) and per-call scratch (clean at every call boundary).
 *
 * File layout, little-endian, format version 1:
 *   header (144 bytes): char magic[8] = "DINTIMG1"; u32 version; u32 kind; dint_cfg cfg, 76 bytes, flags included;
 *     u32 n_regions; u64 kv_capacity[5] (entries of every KV table at save time, 0 past n_tables); u32 tpool_cap (the
 *     eBPF TATP chain pool's entries); u32 n_tables;
 *   n_regions records of 24 bytes: {u32 index; u32 0; u64 raw bytes; u64 blocks = ceil(raw bytes / 64 MiB)};
 *   then the blocks of every region in order.  A region is cut into 64 MiB raw blocks, the last one shorter.  A block
 *   of B raw bytes has L = ceil(B / 128) lines and is stored as:
 *     u32 bitmap[ceil(L / 128) * 4]   bit i of word w = line 32 w + i holds a non-zero byte (padding words are 0);
 *     the lines whose bit is set, in order, 128 bytes each; a partial last line (B % 128 != 0) keeps only its B % 128
 *       in-range bytes;
 *     u64 checksum: the sum mod 2^64 of fasthash64(word, 4 bytes, seed 2 w) over every bitmap word w and
 *       fasthash64(line, 128 bytes zero-padded, seed 2 i + 1) over every stored line i (its index in the block).  The
 *       sum does not depend on the order of the device's reduction; it detects corruption and is no defence against an
 *       attacker.
 */
int dint_image_save(dint_engine *e, const char *path);
int dint_image_open(const char *path, int device, dint_engine **out);
int dint_cluster_image_save(dint_cluster *c, const char *dir);
int dint_cluster_image_open(const char *dir, int n_gpus, const int *devices, uint64_t max_batch, dint_cluster **out);
int dint_image_times(double out[4]);

/*
 * Re-sharding: the state of a lock_2pl, lock_fasst or store cluster does not depend on its shard count G, only its layout
 * over the shards does (shard r owns the lock slots / buckets s with s % G == r, at local index s / G).
 *   dint_cluster_reshard: a new cluster of n_gpus shards holding src's state, which answers every later request exactly
 *     as src would.  src is read, never changed, and stays usable.  It synchronises every source device first (a quiesce
 *     point, like dint_snapshot_create: nothing may be in flight on src), then builds the destination as
 *     dint_cluster_create(kind, cfg, n_gpus, devices, max_batch) would -- same exchange buffers, chunk, slab capacity and
 *     persisting-L2 window, and the same `cfg`, so a later dint_cluster_image_save writes a manifest that
 *     dint_cluster_image_open(dir, n_gpus, ...) accepts -- and fills every shard on its own device:
 *       lock_2pl   {num_ex, num_sh} of every slot;
 *       lock_fasst the version and the lock bit of every slot: a lock granted before the call is still held after it;
 *       store      every live key with its value and version (tombstones are dropped; each destination table is at least
 *                  as large as dint_cluster_create would make it, and large enough to keep its keys at <= 35 % load, so
 *                  the tombstone rehash does not run on the first call); with DINT_CFG_STORE_EBPF_* every 256-byte cache
 *                  set moves whole (keys, versions, valid and dirty masks, bloom word).
 *     A source shard on another GPU is read over peer memory (peer access is enabled for each such pair, DINT_ENODEV
 *     where there is none).  Statistics (dint_stats, the cache tier's counters) start at zero, as after an image open.
 *     Peak device memory is the source plus the destination: destroy src afterwards to release it.
 *     A key that reached a store table twice (a second eBPF kInsert of it) keeps both copies, but which one a lookup
 *     finds may change -- the limit the tombstone rehash already has (DINT_CFG_STORE_EBPF_*, "Limit").
 *     DINT_EINVAL and no cluster (*out = NULL): tatp and smallbank (their shard count is the clients' replica placement,
 *     primary key % G with backups +1 and +2, so another count changes which shard is primary for a key and there is no
 *     one-server state to move), log_server (a record belongs to the rank that received it; no key decides ownership),
 *     n_gpus outside 1..8, and devices that are neither all distinct nor all the same.  n_gpus == G is a plain copy.
 *   dint_reshard_times: the last dint_cluster_reshard of this thread, in seconds: [0] wall, [1] the re-shard kernels
 *     (CUDA events, summed over the destination shards), [2] the key count and the destination engines' allocation.
 */
int dint_cluster_reshard(dint_cluster *src, int n_gpus, const int *devices, uint64_t max_batch, dint_cluster **out);
int dint_reshard_times(double out[3]);

/*
 * Rebuilding lost tatp / smallbank shards from their replicas.
 *   Placement: the engine's own.  A cluster of G shards (G = 1 or 3..8; an engine alone places with
 *     txn_shards > 3 ? txn_shards : 3) keeps the rows of key k on its three replicas, shards (k % G + i) % G of roles
 *     i = 0 (primary), 1 and 2 (backups): the clients write every row there (txn_clients.cuh), and population places
 *     rows the same way, so each shard holds every row of every key it is a replica of.  With G = 3 every shard holds
 *     every key.
 *   Lost set: any set of shards that leaves every key at least one surviving replica -- for G >= 4 no three cyclically
 *     consecutive shards, for G = 3 at most two.  G = 1 has nothing to rebuild from.
 *   Source rule: for each key the source is its surviving replica with the lowest role; that copy (value and version) is
 *     inserted once into every lost replica of the key.  The rule depends on (k, G, lost set) alone, so the result is
 *     deterministic.
 *   Exactness: at a replica-consistent point -- every write served at all of its replicas: after population, or after
 *     traffic made of whole transactions -- a rebuilt shard's rows equal the lost shard's: the same keys in every table,
 *     the same values and versions (kCommitBck bumps a version exactly as kCommitPrim does), and deleted rows absent.
 *   Mid-transaction: the clients commit the log, then the backups, then the primary, in separate rounds.  At a round
 *     boundary the backups can be one write ahead of a primary that still holds that key's lock, and a rebuilt primary
 *     then takes the backups' newer row.
 *   Not rebuilt, because it cannot be: TATP lock words and holder keys, and SmallBank's {num_ex, num_sh} counters, start
 *     free (a lock slot is shared by keys of different primaries, so a peer's slot cannot be attributed to keys); the
 *     log ring starts empty (for G > 3 a shard's arrival order cannot be recovered from its peers, and nothing reads
 *     the log); statistics start at zero, as after an image open.
 *   dint_cluster_rebuild: rebuild the shards of bit mask lost_mask in place.  It synchronises every device (a quiesce
 *     point, as dint_cluster_reshard), builds each lost shard's new engine on that shard's device from the shard's
 *     configuration (its tables at least as large as dint_cluster_create makes them, and large enough to keep their
 *     rows at <= 35 % load) and fills it from the surviving replicas over peer memory; the old engine's state is never
 *     read.  Only then the new engines replace the old ones, and every rank's exchange context is made again over the
 *     cluster's exchange buffers, signal blocks zeroed, as dint_cluster_create makes them.  On any failure the cluster is
 *     left as it was.  Peak device memory: the cluster plus the new engines.
 *     DINT_EINVAL, the cluster unchanged: lock_2pl, lock_fasst, store and log_server clusters (no replicas); G = 1; an
 *     empty mask or one naming shards outside [0, G); a lost set that leaves some key without a replica;
 *     DINT_CFG_TATP_EBPF and DINT_CFG_SMALLBANK_EBPF (their cache tiers hold dirty and cache-only rows whose wire-visible
 *     versions depend on each shard's own hit history); and a cluster with dint_txn_clients attached (clients
 *     mid-transaction hold locks that are lost -- a SmallBank release would drive a counter below zero).
 *   dint_cluster_image_open_rebuild: dint_cluster_image_open, except that a shard image that is missing or fails with
 *     DINT_EIO (short file, I/O error, checksum) is rebuilt from the others, which are opened first.  *rebuilt_mask
 *     receives the shards rebuilt (0: the image was whole).  The manifest must be valid (DINT_EIO when missing), and
 *     DINT_EINVAL from a shard image (foreign kind, flags, layout) stays an error.  A failed set that cannot be rebuilt
 *     (by the rules above) returns DINT_EIO naming the shards; missing files are judged before any CUDA call.  The shard
 *     images of one directory are of one moment (the manifest is written last), so the rebuilt rows are those the lost
 *     shard saved.  To repair a directory, open it this way and save to ANOTHER directory: a save removes the manifest
 *     before it rewrites shards, so an in-place repair that stopped part-way would leave nothing to open.
 *   dint_rebuild_times: the last rebuild of this thread, in seconds: [0] wall, [1] the rebuild kernels (CUDA events,
 *     summed over the lost shards), [2] the row count and the new engines' allocation.
 */
int dint_cluster_rebuild(dint_cluster *c, uint32_t lost_mask);
int dint_cluster_image_open_rebuild(const char *dir, int n_gpus, const int *devices, uint64_t max_batch, uint32_t *rebuilt_mask,
                                    dint_cluster **out);
int dint_rebuild_times(double out[3]);

/*
 * Re-sharding tatp / smallbank clusters: re-placing every row on its replicas under another shard count.
 *   dint_cluster_reshard_txn: a new tatp or smallbank cluster of n_gpus shards (1 or 3..8), built as
 *     dint_cluster_create(kind, src's cfg, n_gpus, devices, max_batch) would build it.  Each shard j holds, for every key
 *     it replicates under the new placement (j is (k % n_gpus + i) % n_gpus for some i in 0..2), the row of the key's
 *     old primary, shard k % G of src: its value and version.  At a drained point (dint_txn_clients_drain, or population
 *     and nothing since) every replica of a key holds the same row, so the new cluster answers every later transaction
 *     as src would under the new placement.  One fixed source per key makes the result independent of launch order.
 *     Only FULL rows move; deleted rows stay absent.  Each table is at least as large as dint_cluster_create makes it,
 *     and large enough to keep its rows at <= 35 % load.
 *     Not moved: lock words, holder keys and SmallBank counters start free (the call requires them free, so nothing is
 *     lost); the log ring starts empty (nothing reads it, and for G > 3 arrival order has no meaning on another shard);
 *     statistics start at zero.  src is read, never changed, and stays usable; it is synchronised first.  A source shard
 *     on another GPU is read over peer memory.  Peak device memory is src plus the new cluster.  The call is timed in
 *     dint_reshard_times.
 *     DINT_EINVAL, *out = NULL and src unchanged, with the reason in dint_last_error(): kinds other than tatp and
 *     smallbank (their call is dint_cluster_reshard); DINT_CFG_TATP_EBPF and DINT_CFG_SMALLBANK_EBPF (as for
 *     dint_cluster_rebuild); n_gpus of 0, 2 or more than 8; devices neither all distinct nor all the same; and any held
 *     lock (a TATP lock bit, a SmallBank counter not {0, 0}) on any source shard, naming the shard and the count: clients
 *     are mid-transaction, drain them first.
 */
int dint_cluster_reshard_txn(dint_cluster *src, int n_gpus, const int *devices, uint64_t max_batch, dint_cluster **out);

/*
 * lock_2pl, lock_fasst, log_server and store closed-loop clients ON the GPU (SURVEY.md section 8(f) rank 2).  The
 * reference's clients are Caladan uthreads on other machines (lock_2pl/caladan/client.cc:181-230,
 * lock_fasst/caladan/client.cc:183-280, store/caladan/client_udp.cc:135-208; trace shapes lock_2pl/caladan/
 * trace_init.sh:9-24, lock_fasst/caladan/trace_init.sh:9-27, log_server/caladan/trace_init.sh:15-19); here n_clients of
 * those state machines live next to the engine, one request outstanding each per round, so committed txn/s and the
 * abort rate are produced live instead of replayed.  The kind is the engine's.  Same decisions, draw for draw, as the
 * host-side clients of dint_b200/csrc/workloads.cc (seed, client id; the store REF family's LCG is seeded with
 * 0xdeadbeef + client index, as the reference's, whatever `seed`).
 *   dint_clients_create_cfg: the workload family, with the fields of dint_wl_cfg.  Reference: 24,000,000 lock ids,
 *     uniform (theta 0), read_pct 80; store: 2,000,000 subscribers, set_pct 0 "parallel" or 50 "contention".  DINT_EINVAL for a tatp / smallbank engine (their clients: dint_txn_clients_*), n_clients == 0,
 *     n_keys == 0 (lock kinds, HOT store), read_pct or set_pct > 100, store_subscribers == 0 (REF store).
 *   dint_clients_create: lock_fasst clients (lock_fasst engine only) of the given family.
 *   dint_clients_run: `rounds` rounds, asynchronous on cuda_stream.
 *   dint_clients_stats (synchronises): requests served, committed transactions, validation aborts, lock rejects, rounds.
 *   dint_clients_stats_all (synchronises): requests served, committed transactions, validation aborts, lock rejects,
 *     not-exist replies (store), rounds: the order of dint_wl_stats.
 *   dint_clients_peek (test hook, synchronises): the next round's requests / the last round's replies,
 *     n_clients * dint_msg_size(kind) bytes.
 */
typedef struct dint_clients_cfg {
  uint32_t n_clients;
  uint32_t n_keys;             /* lock kinds: ids in [0, n_keys); store HOT: hot-set size */
  uint64_t seed;
  double   zipf_theta;         /* 0 = uniform */
  uint32_t read_pct;           /* lock kinds: a key is read-only / shared with this probability (percent) */
  uint32_t set_pct;            /* store: percent of kSet (0 = "parallel", 50 = "contention") */
  uint32_t store_subscribers;  /* store: kSubscriberNum of the key generator */
  uint32_t store_hot;          /* store: 1 = HOT family */
  uint32_t reserved[4];
} dint_clients_cfg;
typedef struct dint_clients dint_clients;
/* kind = the engine's: lock_2pl, lock_fasst, log or store (tatp / smallbank: dint_txn_clients_*) */
int dint_clients_create_cfg(dint_engine *e, const dint_clients_cfg *cfg, dint_clients **out);
int dint_clients_create(dint_engine *e, uint32_t n_clients, uint64_t seed, uint32_t n_keys, double zipf_theta, uint32_t read_pct,
                        dint_clients **out);
int dint_clients_run(dint_clients *c, uint32_t rounds, void *cuda_stream);
int dint_clients_stats(dint_clients *c, uint64_t out[5]);
/* requests, committed, validation aborts, lock rejects, not-exist replies, rounds: the order of dint_wl_stats */
int dint_clients_stats_all(dint_clients *c, uint64_t out[6]);
int dint_clients_peek(dint_clients *c, void *next_req_host, void *last_resp_host);
void dint_clients_destroy(dint_clients *c);

/*
 * TATP and SmallBank closed-loop clients ON the GPU, against a shard cluster (kind and shard count from the cluster:
 * tatp or smallbank, 1 or 3-8 shards).  The state machines are those of the host drivers (TxnWorkload,
 * dint_b200/csrc/txn_clients.cuh is the one statement of both): same draws, same decisions, same records in the same
 * order.  Clients [gid0, gid0 + n_clients) are split over the cluster's ranks in contiguous blocks; `subscribers` is
 * kSubscriberNum (tatp) or kAccountNum (smallbank), as in the host drivers, and must match the servers' population.
 * The cluster must outlive the clients.
 *   dint_txn_clients_run (blocking): `rounds` rounds, each emitted on the devices and served with one exchange step;
 *     one host synchronise per round reads the round's per-(rank, shard) record counts, which size the exchange slabs
 *     exactly.  A round that does not fit the cluster's slabs or batch size is served in pieces (counted in stats[18]).
 *     Returns 0, DINT_EPROTO (an engine answered with an error reply), or an error.
 *   dint_txn_clients_stats: dint_txn_stats' 18 words (requests and rounds SERVED), then rounds served in pieces.
 *   dint_txn_clients_peek (test hook, synchronises): in global client order, the pending round (n_next records and
 *     their destination shards) and the replies absorbed last (n_last records); buffers of n_clients * 9 records.
 *   dint_txn_clients_times: rounds timed by run, their host wall time (s) and the CUDA-event time (s) of their device
 *     work on rank 0's stream; the difference is the host time the round-trip leaves exposed.
 *   dint_txn_clients_drain (blocking): serve rounds in draining mode -- every client finishes the transaction it is in
 *     and starts no new one -- until the pending round is empty.  *rounds receives the rounds served (they count in
 *     stats; no transaction starts during a drain).  A drain ends within L + 1 emissions, L the longest transaction in
 *     rounds (TATP 7, SmallBank 5): at most L rounds served.  Returns 0 when drained, DINT_EPROTO as run does, and
 *     DINT_EINVAL with the count of clients still mid-transaction when records are pending after max_rounds (the
 *     clients then continue at the next run).  Drained clients stay idle until the next run, peek or stats call, which
 *     resumes them: every idle client begins its next transaction and emits on the cluster it is bound to.  Each
 *     client's transaction stream is the one it would have run without the drain, only later.
 *   dint_txn_clients_rebind: move drained clients, or clients that have never emitted, to cluster c (e.g. the result of
 *     dint_cluster_reshard_txn): each client's state moves to c's ranks in contiguous blocks, across devices if needed,
 *     and the counters carry over.  Afterwards the clients no longer reference the old cluster, which may be destroyed:
 *     its dint_txn_clients attachment (the one dint_cluster_rebuild refuses) moves to c.  DINT_EINVAL, the clients
 *     unchanged: clients mid-transaction, a cluster of another kind, and every cluster dint_txn_clients_create refuses.
 * The first round is emitted by the first run, peek or stats call.
 */
typedef struct dint_txn_clients dint_txn_clients;
int dint_txn_clients_create(dint_cluster *c, uint32_t n_clients, uint32_t gid0, uint32_t subscribers, dint_txn_clients **out);
int dint_txn_clients_run(dint_txn_clients *t, uint32_t rounds);
int dint_txn_clients_stats(dint_txn_clients *t, uint64_t out[19]);
int dint_txn_clients_peek(dint_txn_clients *t, void *next_req, uint8_t *next_dst, uint64_t *n_next, void *last_resp, uint64_t *n_last);
int dint_txn_clients_times(dint_txn_clients *t, double out[3]);
int dint_txn_clients_drain(dint_txn_clients *t, uint32_t max_rounds, uint32_t *rounds);
int dint_txn_clients_rebind(dint_txn_clients *t, dint_cluster *c);
/* The lock counters of tatp/caladan/client_lock.cc, summed over the clients (synchronises): [0] kAcquireLock replies
 * absorbed (lock_cnt, :718,1056,1309,1583), [1] of them kRejectLock = refused through false sharing
 * (reject_sharing_cnt), [2] kRejectLockSameKey = refused by a holder of the same key (reject_same_key_cnt); the two
 * ratios [1]/[0] and [2]/[0] are what the reference prints (:403-428,449-462).  [2] stays 0 against servers without
 * DINT_CFG_LOCK_HOLDER_KEYS; smallbank: all 0 (S/X counters have no single holder, and no such wire type).  The host
 * clients of libdint_wl.so count the same three words. */
int dint_txn_clients_lock_stats(dint_txn_clients *t, uint64_t out[3]);
void dint_txn_clients_destroy(dint_txn_clients *t);

/*
 * lock_2pl, lock_fasst, store and log_server closed-loop clients ON the GPU, against a shard cluster: the clients of
 * dint_clients_create_cfg (same family fields, same draws and decisions), with the kind and shard count taken from the
 * cluster.  Clients [0, n_clients) are split over the ranks in contiguous blocks, rank r's block on rank r's device (a
 * rank may hold none).  A cluster of these kinds answers like ONE sequential server fed the rank-major concatenation, so
 * the clients send and absorb, round for round, exactly what dint_clients with the same clients on one engine would.
 * The cluster must outlive the clients.
 *   dint_cluster_clients_create: DINT_EINVAL for a tatp / smallbank cluster (their clients: dint_txn_clients_*), for
 *     every argument dint_clients_create_cfg refuses, and when a rank's block (n_clients / shards, rounded up) exceeds
 *     the cluster's max_batch -- every round would then be served in pieces.
 *   dint_cluster_clients_run (blocking): `rounds` rounds.  Each rank's clients emit one record each and a kernel counts
 *     them per owner shard; one host synchronise per round reads the counts, which size the exchange slabs exactly, and
 *     one exchange step serves the round.  A round whose largest (rank, shard) count exceeds the cluster's slab capacity
 *     is served one source rank at a time, in pieces (counted in stats[6]).  log_server rounds skip the exchange (a log
 *     record is owned by the rank that received it): each rank's engine serves its own batch.  Returns 0, DINT_EPROTO
 *     (an engine answered with an error reply), or an error.
 *   dint_cluster_clients_stats (synchronises): dint_clients_stats_all's 6 words (rounds counted once, not per rank),
 *     then rounds served in pieces.
 *   dint_cluster_clients_peek (test hook, synchronises): in global client order, the next round's requests / the last
 *     round's replies, n_clients * dint_msg_size(kind) bytes each.
 *   dint_cluster_clients_times: as dint_txn_clients_times.
 *   dint_cluster_clients_rebind: move the clients to cluster c (e.g. the result of dint_cluster_reshard): their state,
 *     the pending round's requests and the last replies are redistributed over c's ranks in contiguous blocks, across
 *     devices if needed, and the counters carry over, so stats keep counting from where they were.  Afterwards the
 *     clients no longer reference the old cluster, which may be destroyed.  DINT_EINVAL (the clients unchanged) for a
 *     cluster of another kind, and when a rank's block of c exceeds c's max_batch, as at create.
 * The first round is emitted by the first run or peek call.
 */
typedef struct dint_cluster_clients dint_cluster_clients;
int dint_cluster_clients_create(dint_cluster *c, const dint_clients_cfg *cfg, dint_cluster_clients **out);
int dint_cluster_clients_run(dint_cluster_clients *t, uint32_t rounds);
int dint_cluster_clients_stats(dint_cluster_clients *t, uint64_t out[7]);
int dint_cluster_clients_peek(dint_cluster_clients *t, void *next_req, void *last_resp);
int dint_cluster_clients_times(dint_cluster_clients *t, double out[3]);
int dint_cluster_clients_rebind(dint_cluster_clients *t, dint_cluster *c);
void dint_cluster_clients_destroy(dint_cluster_clients *t);

int dint_get_stats(dint_engine *e, dint_stats *s);
void dint_reset_stats(dint_engine *e);
/* per-kernel CUDA-event timing: 0 = off, 1 = every kernel, otherwise a bit mask over
 * {1<<0 k_classify, 1<<1 k_log_scan, 1<<2 k_apply, 1<<3 k_ordered, 1<<4 k_kv_load} */
int dint_profile(dint_engine *e, int enable);
int dint_kernel_times(dint_engine *e, dint_kernel_time *out, int max_entries);  /* returns #entries */
const char *dint_last_error(void);

/* pinned host memory for req/resp buffers */
void *dint_host_alloc(size_t bytes);
void dint_host_free(void *p);

/* hooks for unit tests of the host/device-shared arithmetic (no GPU needed) */
uint64_t dint_test_fasthash64(uint64_t x, int len);      /* len 4 or 8, seed 0xdeadbeef */
uint32_t dint_test_fastmod(uint64_t n, uint32_t d);
/* the source shard dint_cluster_rebuild copies key's rows from in a G-shard cluster that lost the shards of lost_mask,
 * or -1 when every replica of the key is lost (or G is outside 1..8) */
int dint_test_rebuild_source(uint64_t key, uint32_t G, uint32_t lost_mask);
/* the bit mask of shards dint_cluster_reshard_txn gives key's row when it re-places a G-shard cluster onto G2 shards and
 * reads source shard src: (k % G2 + i) % G2 for i = 0..2 when src == k % G, else 0 (0 also for G or G2 outside 1..8) */
uint32_t dint_test_txn_reshard_dests(uint64_t key, uint32_t G, uint32_t G2, uint32_t src);
/* test hook: the slice sizes dint_submit cuts a call of n requests into (host logic, no GPU needed);
 * returns the number of slices, writes the first `cap` of them */
uint32_t dint_test_host_slices(uint64_t n, uint32_t min_slice, uint32_t max_slice, int ramp_up, uint32_t *out, uint32_t cap);

#ifdef __cplusplus
}
#endif
#endif
