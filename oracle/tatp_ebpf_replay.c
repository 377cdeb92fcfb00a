/* oracle/tatp_ebpf_replay.c -- TEST INFRASTRUCTURE.  Replays a trace through the reference's eBPF TATP shard server,
 * built from its unmodified sources (oracle/tatp_ebpf.mk links tatp/ebpf/shard_kern.c or lock_kern.c, compiled as
 * user-space C against oracle/ebpf_shim, and includes tatp/ebpf/kvs.h).  One request at a time, as one server thread:
 *   XDP (tps_prim_xdp_main) -> XDP_TX: the reply leaves as it is;
 *                           -> XDP_PASS: the user-space dispatch below (restated from shard_user.c:171-247, which
 *                              lock_user.c repeats), then TC egress (tps_prim_tc_main) on the 108-byte reply.  TC
 *                              shrinks it back to struct message, except after COMMIT_BCK_ACK (shard_kern.c:1231): that
 *                              reply leaves as ext_message, whose first 55 bytes are what is written here.
 * A request the user-space dispatch panics on (a type it does not know, a READ / COMMIT / INSERT that XDP did not extend,
 * which is what a table >= 5 gives) is written with type 0xFF, and so is a DELETE of table >= 5 (kvs_delete would index
 * tables[] out of bounds).
 *
 * usage: tatp_ebpf_{shard,lock} REQ RESP [--populate S] [--shard I] [--dump KEYS SETS CHAINS FINDS LOCKS LOG]
 *   REQ / RESP: n packed 55-byte struct message.  --populate S first serves the eBPF client's population stream for S
 *   subscribers as shard I of three sees it (tatp/caladan/client_ebpf_shard.cc:96-339: 600 populate threads in thread
 *   order, fastrand restarting at 0xdeadbeef per thread; kInsertPrim where key % 3 == I, kInsertBck otherwise; bytes the
 *   client leaves uninitialised are zero).
 *   KEYS: n x {u64 key; u64 table}.  Per key: SETS gets the 232-byte struct cache_entry of its bucket; CHAINS gets
 *   {u32 n; 8 x {u64 key[4]; u32 ver[4]; u8 valid[4]; u8 val[4][40]}} (the bucket's chain head first, n entries, the rest
 *   zero); FINDS gets {u32 found; u32 ver; u8 val[40]} (kvs_get); LOCKS gets {u64 lock_bit; u64 holder} of its lock slot
 *   (holder 0 for shard_kern.c).  LOG gets the first min(appends, MAX_LOG_ENTRY_NUM) 64-byte struct log_entry. */
#define _GNU_SOURCE
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <arpa/inet.h>
#include <linux/bpf.h>
#include <linux/ip.h>
#include <linux/udp.h>
#include <linux/if_ether.h>
#include <linux/pkt_cls.h>

static volatile int quit = 0;   /* utils.h's panic() sets it */
#include "utils.h"
#include "kvs.h"

int tps_prim_xdp_main(struct xdp_md *ctx);
int tps_prim_tc_main(struct __sk_buff *skb);

#ifndef TATP_EBPF_LOCK
#define TATP_EBPF_LOCK 0
#endif

/* the programs' maps, defined (as anonymous struct types) in the kernel program */
extern char map_locks_sub, map_locks_sec_sub, map_locks_ai, map_locks_sf, map_locks_cf;
extern char map_cache_sub, map_cache_sec_sub, map_cache_ai, map_cache_sf, map_cache_cf;
extern char map_log;
static const void *lock_maps[TABLE_NUM] = {&map_locks_sub, &map_locks_sec_sub, &map_locks_ai, &map_locks_sf, &map_locks_cf};
static const void *cache_maps[TABLE_NUM] = {&map_cache_sub, &map_cache_sec_sub, &map_cache_ai, &map_cache_sf, &map_cache_cf};
static const uint32_t hash_size[TABLE_NUM] = {SUB_HASH_SIZE, SEC_SUB_HASH_SIZE, AI_HASH_SIZE, SF_HASH_SIZE, CF_HASH_SIZE};

/* ---- bpf_map_lookup_elem of the shim: one lazily allocated zeroed array per map (12 maps are looked up) ----------- */
enum { NMAPS = 16 };
static struct { const void *map; uint8_t *base; size_t vsz, n; } maps[NMAPS];
void *shim_map_lookup(const void *map, size_t value_size, size_t max_entries, uint32_t key) {
  int i = 0;
  for (; i < NMAPS && maps[i].map && maps[i].map != map; i++) {}
  if (i == NMAPS) { fprintf(stderr, "too many maps\n"); exit(2); }
  if (!maps[i].map) {
    maps[i].map = map;
    maps[i].vsz = value_size;
    maps[i].n = max_entries;
    maps[i].base = calloc(max_entries, value_size);
    if (!maps[i].base) { fprintf(stderr, "map allocation failed\n"); exit(2); }
  }
  if (key >= maps[i].n) return NULL;
  return maps[i].base + (size_t)key * maps[i].vsz;
}
static const uint8_t *map_elem(const void *map, uint32_t key) {   /* NULL: no request ever looked the map up */
  for (int i = 0; i < NMAPS && maps[i].map; i++)
    if (maps[i].map == map) return key < maps[i].n ? maps[i].base + (size_t)key * maps[i].vsz : NULL;
  return NULL;
}

static struct kvs *tables[TABLE_NUM];
static uint64_t log_appends;

/* The bloom word user space sends back after a delete (restating shard_user.c:94-104): for every entry of the bucket's
 * chain, the bit picked by the top six bits of fasthash64 over the entry's whole 32-byte key array. */
static uint64_t chain_bloom_word(uint8_t t, uint32_t bucket) {
  uint64_t word = 0;
  for (const struct kvs_entry *ent = tables[t]->bucket_heads[bucket]; ent != NULL; ent = ent->next)
    word |= (uint64_t)1 << (fasthash64(ent->key, KEYS_PER_ENTRY * sizeof(uint64_t), 0xdeadbeef) >> 58);
  return word;
}

static uint8_t *pkt;                 /* below 4 GB: xdp_md / __sk_buff hold packet addresses in __u32 */
enum { HDR = sizeof(struct ethhdr) + sizeof(struct iphdr) + sizeof(struct udphdr) };

static void headers(uint16_t sport, uint16_t dport, size_t payload) {
  memset(pkt, 0, HDR);
  struct iphdr *ip = (struct iphdr *)(pkt + sizeof(struct ethhdr));
  ip->ihl = 5; ip->version = 4;
  ip->tot_len = htons((uint16_t)(sizeof(struct iphdr) + sizeof(struct udphdr) + payload));
  struct udphdr *udp = (struct udphdr *)(pkt + sizeof(struct ethhdr) + sizeof(struct iphdr));
  udp->source = htons(sport); udp->dest = htons(dport);
  udp->len = htons((uint16_t)(sizeof(struct udphdr) + payload));
}

/* one request in, the first 55 bytes of its reply out */
static void serve(const struct message *req, struct message *reply) {
  headers(40000, FASST_PORT, sizeof(struct message));
  memset(pkt + HDR, 0, sizeof(struct ext_message));
  memcpy(pkt + HDR, req, sizeof *req);
  struct xdp_md ctx;
  memset(&ctx, 0, sizeof ctx);
  ctx.data = (uint32_t)(uintptr_t)pkt;
  ctx.data_end = ctx.data + HDR + sizeof(struct message);
  if (tps_prim_xdp_main(&ctx) == XDP_TX) {
    memcpy(reply, pkt + HDR, sizeof *reply);
    if (reply->type == COMMIT_LOG_ACK || reply->type == DELETE_LOG_ACK) log_appends++;
    return;
  }
  const size_t ret = ctx.data_end - ctx.data - HDR;
  struct ext_message msg;
  memset(&msg, 0, sizeof msg);
  memcpy(&msg, pkt + HDR, ret < sizeof msg ? ret : sizeof msg);
  const int ext = ret == sizeof(struct ext_message);
  int ok = msg.table < TABLE_NUM;
  /* ---- shard_user.c:171-247 ---- */
  if (ok && msg.type == READ && ext) {
    if (msg.ver1 == 1) kvs_set(tables[msg.table], msg.key2, msg.val2, msg.ver2);
    int res = kvs_get(tables[msg.table], msg.key1, msg.val1, &msg.ver1);
    msg.type = res == 0 ? GRANT_READ : NOT_EXIST;
  } else if (ok && (msg.type == COMMIT_PRIM || msg.type == COMMIT_BCK) && ext) {
    if (msg.ver1 == 1) kvs_set(tables[msg.table], msg.key2, msg.val2, msg.ver2);
    msg.ver1 = kvs_set(tables[msg.table], msg.key1, msg.val1, 0);
    msg.type = msg.type == COMMIT_PRIM ? COMMIT_PRIM_ACK : COMMIT_BCK_ACK;
  } else if (ok && (msg.type == INSERT_PRIM || msg.type == INSERT_BCK) && ext) {
    kvs_insert(tables[msg.table], msg.key1, msg.val1);
    kvs_set(tables[msg.table], msg.key2, msg.val2, msg.ver2);
    msg.type = msg.type == INSERT_PRIM ? INSERT_PRIM_ACK : INSERT_BCK_ACK;
  } else if (ok && (msg.type == DELETE_PRIM || msg.type == DELETE_BCK) && ret == sizeof(struct message)) {
    kvs_delete(tables[msg.table], msg.key1);
    const uint64_t word = chain_bloom_word(msg.table, kvs_hash(tables[msg.table], msg.key1));
    memcpy(msg.val1, &word, sizeof word);           /* the first 8 value bytes carry it */
    msg.type = msg.type == DELETE_PRIM ? DELETE_PRIM_ACK : DELETE_BCK_ACK;
  } else {
    memcpy(reply, req, sizeof *reply);
    reply->type = 0xFF;
    return;
  }
  /* ---- the reply through TC egress ---- */
  headers(FASST_PORT, 40000, sizeof msg);
  memcpy(pkt + HDR, &msg, sizeof msg);
  struct __sk_buff skb;
  memset(&skb, 0, sizeof skb);
  skb.data = (uint32_t)(uintptr_t)pkt;
  skb.len = HDR + sizeof msg;
  skb.data_end = skb.data + skb.len;
  tps_prim_tc_main(&skb);
  memcpy(reply, pkt + HDR, sizeof *reply);
}

static void *slurp(const char *path, size_t *len) {
  FILE *f = fopen(path, "rb");
  if (!f) { perror(path); exit(2); }
  fseek(f, 0, SEEK_END);
  *len = (size_t)ftell(f);
  fseek(f, 0, SEEK_SET);
  void *p = malloc(*len ? *len : 1);
  if (*len && fread(p, 1, *len, f) != *len) { perror(path); exit(2); }
  fclose(f);
  return p;
}
static FILE *wopen(const char *path) {
  FILE *f = fopen(path, "wb");
  if (!f) { perror(path); exit(2); }
  return f;
}

/* ---- population (tatp/caladan/client_ebpf_shard.cc:96-339) ---------------------------------------------------- */
static uint32_t shard_of_me;
static uint32_t fastrand(uint64_t *seed) {   /* tatp/caladan/tatp.h:32-35 */
  *seed = *seed * 1103515245 + 12345;
  return (uint32_t)(*seed >> 32);
}
static int select_types(uint64_t *seed, uint8_t out[4]) {   /* tatp.h:254-280 with values {1,2,3,4}, N = 1, M = 4 */
  int used[8] = {0}, n = (int)(fastrand(seed) % 4) + 1;
  for (int i = 0; i < n; i++) {
    uint8_t v = (uint8_t)(fastrand(seed) % 4 + 1);
    if (used[v]) { i--; continue; }
    used[v] = 1;
    out[i] = v;
  }
  return n;
}
static uint64_t sub_nbr(uint32_t s) {   /* tatp_sid_to_sub_nbr: 3 x 12-bit BCD groups */
  uint64_t r = 0;
  for (int g = 0; g < 3; g++, s /= 1000) {
    uint32_t i = s % 1000;
    r |= (uint64_t)(((i / 100) % 10) << 8 | ((i / 10) % 10) << 4 | (i % 10)) << (12 * g);
  }
  return r;
}
static void pop_row(uint8_t table, uint64_t key, const uint8_t *val) {
  struct message msg, reply;
  memset(&msg, 0, sizeof msg);
  msg.type = key % 3 == shard_of_me ? INSERT_PRIM : INSERT_BCK;
  msg.table = table;
  msg.key = key;
  memcpy(msg.val, val, VAL_SIZE);
  serve(&msg, &reply);
}
static void populate(uint32_t S) {
  const uint32_t threads = 600, slice = S / threads;
  for (uint32_t w = 0; w < threads; w++) {
    uint64_t seed = 0xdeadbeef;
    const uint32_t lo = w * slice, hi = (w == threads - 1) ? S : (w + 1) * slice;
    uint8_t v[VAL_SIZE];
    for (uint32_t s = lo; s < hi; s++) {                       /* subscriber */
      memset(v, 0, sizeof v);
      uint64_t nbr = sub_nbr(s);
      memcpy(v, &nbr, 8);
      for (int i = 0; i < 5; i++) v[15 + i] = (uint8_t)fastrand(&seed);
      for (int i = 0; i < 10; i++) v[20 + i] = (uint8_t)fastrand(&seed);
      uint16_t bits = (uint16_t)fastrand(&seed);
      memcpy(v + 30, &bits, 2);
      uint32_t msc = 97, vlr = fastrand(&seed);
      memcpy(v + 32, &msc, 4); memcpy(v + 36, &vlr, 4);
      pop_row(SUBSCRIBER, s, v);
    }
    for (uint32_t s = lo; s < hi; s++) {                       /* secondary subscriber */
      memset(v, 0, sizeof v);
      memcpy(v, &s, 4);
      v[4] = 98;
      pop_row(SECOND_SUBSCRIBER, sub_nbr(s), v);
    }
    for (uint32_t s = lo; s < hi; s++) {                       /* access info */
      uint8_t ty[4];
      int n = select_types(&seed, ty);
      for (int i = 0; i < n; i++) {
        memset(v, 0, sizeof v);
        v[0] = 99;
        pop_row(ACCESS_INFO, (uint64_t)s | ((uint64_t)ty[i] << 32), v);
      }
    }
    for (uint32_t s = lo; s < hi; s++) {                       /* special facility + call forwarding */
      uint8_t ty[4];
      int n = select_types(&seed, ty);
      for (int i = 0; i < n; i++) {
        memset(v, 0, sizeof v);
        v[3] = 100;
        v[0] = (fastrand(&seed) % 100 < 85) ? 1 : 0;
        pop_row(SPECIAL_FACILITY, (uint64_t)s | ((uint64_t)ty[i] << 32), v);
        for (uint64_t st = 0; st <= 16; st += 8) {
          if (fastrand(&seed) % 2 == 0) continue;
          memset(v, 0, sizeof v);
          v[1] = 101;
          v[0] = (uint8_t)(fastrand(&seed) % 24 + 1);
          pop_row(CALL_FORWARDING, (uint64_t)s | ((uint64_t)ty[i] << 32) | (st << 40), v);
        }
      }
    }
  }
}

static void dump(const char **p) {
  size_t len = 0;
  uint64_t *kt = slurp(p[0], &len);
  const size_t nk = len / 16;
  FILE *fs = wopen(p[1]), *fc = wopen(p[2]), *ff = wopen(p[3]), *fl = wopen(p[4]);
  for (size_t i = 0; i < nk; i++) {
    const uint64_t key = kt[2 * i];
    const uint8_t t = (uint8_t)kt[2 * i + 1];
    if (t >= TABLE_NUM) { fprintf(stderr, "bad table\n"); exit(2); }
    const uint64_t h = fasthash64(&key, 8, 0xdeadbeef);
    const uint32_t b = (uint32_t)(h % hash_size[t]);
    static const uint8_t zero[sizeof(struct cache_entry)];
    const uint8_t *ce = map_elem(cache_maps[t], b);
    fwrite(ce ? ce : zero, sizeof(struct cache_entry), 1, fs);
    struct { uint64_t key[4]; uint32_t ver[4]; uint8_t valid[4]; uint8_t val[4][VAL_SIZE]; } __attribute__((packed)) rec[8];
    memset(rec, 0, sizeof rec);
    uint32_t n = 0;
    for (struct kvs_entry *e = tables[t]->bucket_heads[b]; e; e = e->next, n++) {
      if (n == 8) { fprintf(stderr, "chain longer than 8 entries\n"); exit(2); }
      memcpy(rec[n].key, e->key, sizeof e->key);
      memcpy(rec[n].ver, e->ver, sizeof e->ver);
      memcpy(rec[n].valid, e->valid, sizeof e->valid);
      memcpy(rec[n].val, e->val, sizeof e->val);
    }
    fwrite(&n, 4, 1, fc);
    fwrite(rec, sizeof rec, 1, fc);
    struct { uint32_t found, ver; uint8_t val[VAL_SIZE]; } fd;
    memset(&fd, 0, sizeof fd);
    fd.found = kvs_get(tables[t], key, fd.val, &fd.ver) == 0;
    fwrite(&fd, sizeof fd, 1, ff);
    uint64_t lk[2] = {0, 0};
    const uint8_t *lw = map_elem(lock_maps[t], (uint32_t)(h % ((uint64_t)hash_size[t] * KEYS_PER_ENTRY)));
    if (lw) memcpy(lk, lw, TATP_EBPF_LOCK ? 16 : 8);
    fwrite(lk, sizeof lk, 1, fl);
  }
  fclose(fs); fclose(fc); fclose(ff); fclose(fl);
  FILE *fg = wopen(p[5]);
  const uint64_t nl = log_appends < MAX_LOG_ENTRY_NUM ? log_appends : MAX_LOG_ENTRY_NUM;
  for (uint64_t i = 0; i < nl; i++) fwrite(map_elem(&map_log, (uint32_t)i), sizeof(struct log_entry), 1, fg);
  fclose(fg);
}

int main(int argc, char **argv) {
  uint32_t pop = 0;
  const char *pos[2] = {0}, *dumps[6] = {0};
  int np = 0, nd = 0;
  for (int i = 1; i < argc; i++) {
    if (!strcmp(argv[i], "--populate") && i + 1 < argc) pop = (uint32_t)strtoul(argv[++i], NULL, 0);
    else if (!strcmp(argv[i], "--shard") && i + 1 < argc) shard_of_me = (uint32_t)strtoul(argv[++i], NULL, 0);
    else if (!strcmp(argv[i], "--dump") && i + 6 < argc) { for (nd = 0; nd < 6; nd++) dumps[nd] = argv[++i]; }
    else if (np < 2) pos[np++] = argv[i];
    else np = 3;
  }
  if (np != 2) {
    fprintf(stderr, "usage: %s REQ RESP [--populate S] [--shard I] [--dump KEYS SETS CHAINS FINDS LOCKS LOG]\n", argv[0]);
    return 2;
  }
  pkt = mmap(NULL, 4096, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_32BIT, -1, 0);
  if (pkt == MAP_FAILED) { perror("mmap"); return 2; }
  for (int t = 0; t < TABLE_NUM; t++) {   /* shard_user.c:83-92 */
    tables[t] = calloc(1, sizeof(struct kvs));
    kvs_init(tables[t], hash_size[t]);
  }
  if (pop) populate(pop);
  size_t len = 0;
  struct message *req = slurp(pos[0], &len);
  const size_t n = len / sizeof(struct message);
  FILE *out = wopen(pos[1]);
  for (size_t i = 0; i < n; i++) {
    struct message reply;
    serve(&req[i], &reply);
    fwrite(&reply, sizeof reply, 1, out);
  }
  fclose(out);
  if (nd == 6) dump(dumps);
  return 0;
}
