/* oracle/smallbank_ebpf_replay.c -- TEST INFRASTRUCTURE.  Replays a trace through the reference's eBPF SmallBank shard
 * server, built from its unmodified sources (oracle/smallbank_ebpf.mk links smallbank/ebpf/shard_kern.c, compiled as
 * user-space C against oracle/ebpf_shim, and includes smallbank/ebpf/kvs.h).  One request at a time, as one server
 * thread:
 *   XDP (tps_prim_xdp_main) -> XDP_TX: the reply leaves as it is;
 *                           -> XDP_PASS: the user-space dispatch below (restated from shard_user.c:139-189), then TC
 *                              egress (tps_prim_tc_main), which installs the answer and shrinks the reply back to the
 *                              23-byte struct message.
 * A request the user-space dispatch panics on is written with type 0xFF and skips TC: a request XDP did not extend (a
 * type outside XDP's list, a table >= 2 on a type other than COMMIT_LOG) fails shard_user.c:142's size check, and a key
 * the table lacks makes kvs_get / kvs_set panic.  The reference's server stops there; here the trace goes on, with what
 * happened before the panic kept (a lock counter's increment, a dirty victim's write-back) and the two locks the panic
 * left held released: the cache set's (XDP takes it for the miss, TC would release it) and the kvs bucket's spin lock.
 *
 * usage: smallbank_ebpf REQ RESP [--populate A] [--warmup] [--shard I] [--shards G] [--dump KEYS SETS FINDS LOCKS LOG]
 *   REQ / RESP: n packed 23-byte struct message.  --populate A first inserts accounts [0, A) into both tables with the
 *   values smallbank.h writes (shard_user.c:70-78; A = ACCOUNT_NUM runs the header's own loop).  --warmup then serves
 *   the eBPF client's warm-up stream as shard I of G sees it (smallbank/caladan/client_ebpf_shard.cc:88-169: for every
 *   account a < A it replicates -- all of them when G <= 3, a % G in {I, I - 1, I - 2} otherwise -- ascending, WARMUP_READ
 *   of (saving, a) then (checking, a)).
 *   KEYS: n x {u64 key; u64 table}.  Per key: SETS gets the 96-byte struct cache_entry of its bucket; FINDS gets
 *   {u32 found; u32 ver; u8 val[8]} (kvs_get's search, without its panic); LOCKS gets the 16-byte struct lock_unit of its
 *   lock slot.  LOG gets the first min(appends, MAX_LOG_ENTRY_NUM) 32-byte struct log_entry. */
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

volatile int quit = 0;   /* utils.h's panic() sets it */
#include "utils.h"
#include "kvs.h"
#include "smallbank.h"

int tps_prim_xdp_main(struct xdp_md *ctx);
int tps_prim_tc_main(struct __sk_buff *skb);

/* the programs' maps, defined (as anonymous struct types) in the kernel program */
extern char map_locks_sav, map_locks_chk, map_cache_sav, map_cache_chk, map_log;
static const void *lock_maps[TABLE_NUM] = {&map_locks_sav, &map_locks_chk};
static const void *cache_maps[TABLE_NUM] = {&map_cache_sav, &map_cache_chk};
static const uint32_t hash_size[TABLE_NUM] = {SAV_HASH_SIZE, CHK_HASH_SIZE};

/* ---- bpf_map_lookup_elem of the shim: one lazily allocated zeroed array per map --------------------------------- */
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
static uint8_t *map_elem(const void *map, uint32_t key) {   /* NULL: no request ever looked the map up */
  for (int i = 0; i < NMAPS && maps[i].map; i++)
    if (maps[i].map == map) return key < maps[i].n ? maps[i].base + (size_t)key * maps[i].vsz : NULL;
  return NULL;
}

static struct kvs *tables[TABLE_NUM];
static uint64_t log_appends;

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

/* one request in, its 23-byte reply out */
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
    if (reply->type == COMMIT_LOG_ACK) log_appends++;
    return;
  }
  const size_t ret = ctx.data_end - ctx.data - HDR;
  struct ext_message msg;
  memset(&msg, 0, sizeof msg);
  memcpy(&msg, pkt + HDR, ret < sizeof msg ? ret : sizeof msg);
  const int ok = ret == sizeof(struct ext_message) && msg.table < TABLE_NUM &&
                 (msg.type == ACQUIRE_SHARED || msg.type == ACQUIRE_EXCLUSIVE || msg.type == COMMIT_PRIM ||
                  msg.type == COMMIT_BCK || msg.type == WARMUP_READ);
  if (!ok) {                                       /* shard_user.c:142 / :188 panic */
    memcpy(reply, req, sizeof *reply);
    reply->type = 0xFF;
    return;
  }
  /* ---- shard_user.c:144-186 ---- */
  quit = 0;
  struct kvs *t = tables[msg.table];
  if (msg.ver1 == 1) kvs_set(t, msg.key2, msg.val2, msg.ver2);
  if (msg.type == COMMIT_PRIM || msg.type == COMMIT_BCK) {
    msg.ver1 = kvs_set(t, msg.key1, msg.val1, 0);
    msg.type = msg.type == COMMIT_PRIM ? COMMIT_PRIM_ACK : COMMIT_BCK_ACK;
  } else {
    kvs_get(t, msg.key1, msg.val1, &msg.ver1);
    msg.type = msg.type == ACQUIRE_SHARED ? GRANT_SHARED : msg.type == ACQUIRE_EXCLUSIVE ? GRANT_EXCLUSIVE : WARMUP_READ_ACK;
  }
  if (quit) {                                      /* a key the table lacks: kvs_get / kvs_set panicked */
    quit = 0;
    t->locks[kvs_hash(t, msg.key1)] = 0;
    const uint64_t h = fasthash64(&msg.key1, sizeof msg.key1, 0xdeadbeef);
    struct cache_entry *e = (struct cache_entry *)map_elem(cache_maps[msg.table], (uint32_t)(h % hash_size[msg.table]));
    if (e) e->lock = 0;
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

/* shard_user.c:70-78 for accounts [0, A): populate_saving_and_checking_tables (smallbank.h:44-66) restated for a prefix */
static void populate(uint32_t A) {
  if (A == ACCOUNT_NUM) { populate_saving_and_checking_tables(tables[SAVING], tables[CHECKING]); return; }
  for (uint32_t a = 0; a < A; a++) {
    struct sb_sav_val_t sv = {sb_sav_magic, 1000000000ull};
    kvs_insert(tables[SAVING], (uint64_t)a, (uint8_t *)&sv);
    struct sb_chk_val_t cv = {sb_chk_magic, 1000000000ull};
    kvs_insert(tables[CHECKING], (uint64_t)a, (uint8_t *)&cv);
  }
}

static void warmup(uint32_t A, uint32_t shard, uint32_t G) {
  for (uint32_t a = 0; a < A; a++) {
    if (G > 3 && (shard + G - a % G) % G > 2) continue;   /* not one of a's primary and two backups */
    for (uint8_t t = 0; t < TABLE_NUM; t++) {
      struct message msg, reply;
      memset(&msg, 0, sizeof msg);
      msg.type = WARMUP_READ;
      msg.table = t;
      msg.key = a;
      serve(&msg, &reply);
    }
  }
}

static void dump(const char **p) {
  size_t len = 0;
  uint64_t *kt = slurp(p[0], &len);
  const size_t nk = len / 16;
  FILE *fs = wopen(p[1]), *ff = wopen(p[2]), *fl = wopen(p[3]);
  for (size_t i = 0; i < nk; i++) {
    const uint64_t key = kt[2 * i];
    const uint8_t t = (uint8_t)kt[2 * i + 1];
    if (t >= TABLE_NUM) { fprintf(stderr, "bad table\n"); exit(2); }
    const uint64_t h = fasthash64(&key, 8, 0xdeadbeef);
    const uint32_t b = (uint32_t)(h % hash_size[t]);
    static const uint8_t zero[sizeof(struct cache_entry)];
    const uint8_t *ce = map_elem(cache_maps[t], b);
    fwrite(ce ? ce : zero, sizeof(struct cache_entry), 1, fs);
    struct { uint32_t found, ver; uint8_t val[VAL_SIZE]; } fd;
    memset(&fd, 0, sizeof fd);
    for (struct kvs_entry *e = tables[t]->bucket_heads[b]; e && !fd.found; e = e->next)   /* kvs.h:40-51 */
      for (int s = 0; s < KEYS_PER_ENTRY; s++)
        if (e->key[s] == key && e->valid[s]) {
          fd.found = 1;
          fd.ver = e->ver[s];
          memcpy(fd.val, e->val[s], VAL_SIZE);
          break;
        }
    fwrite(&fd, sizeof fd, 1, ff);
    static const uint8_t zl[sizeof(struct lock_unit)];
    const uint8_t *lu = map_elem(lock_maps[t], (uint32_t)(h % ((uint64_t)hash_size[t] * KEYS_PER_ENTRY)));
    fwrite(lu ? lu : zl, sizeof(struct lock_unit), 1, fl);
  }
  fclose(fs); fclose(ff); fclose(fl);
  FILE *fg = wopen(p[4]);
  const uint64_t nl = log_appends < MAX_LOG_ENTRY_NUM ? log_appends : MAX_LOG_ENTRY_NUM;
  for (uint64_t i = 0; i < nl; i++) fwrite(map_elem(&map_log, (uint32_t)i), sizeof(struct log_entry), 1, fg);
  fclose(fg);
}

int main(int argc, char **argv) {
  uint32_t pop = 0, shard = 0, G = 3;
  int warm = 0;
  const char *pos[2] = {0}, *dumps[5] = {0};
  int np = 0, nd = 0;
  for (int i = 1; i < argc; i++) {
    if (!strcmp(argv[i], "--populate") && i + 1 < argc) pop = (uint32_t)strtoul(argv[++i], NULL, 0);
    else if (!strcmp(argv[i], "--warmup")) warm = 1;
    else if (!strcmp(argv[i], "--shard") && i + 1 < argc) shard = (uint32_t)strtoul(argv[++i], NULL, 0);
    else if (!strcmp(argv[i], "--shards") && i + 1 < argc) G = (uint32_t)strtoul(argv[++i], NULL, 0);
    else if (!strcmp(argv[i], "--dump") && i + 5 < argc) { for (nd = 0; nd < 5; nd++) dumps[nd] = argv[++i]; }
    else if (np < 2) pos[np++] = argv[i];
    else np = 3;
  }
  if (np != 2 || pop > ACCOUNT_NUM) {
    fprintf(stderr, "usage: %s REQ RESP [--populate A] [--warmup] [--shard I] [--shards G] [--dump KEYS SETS FINDS LOCKS LOG]\n", argv[0]);
    return 2;
  }
  pkt = mmap(NULL, 4096, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_32BIT, -1, 0);
  if (pkt == MAP_FAILED) { perror("mmap"); return 2; }
  for (int t = 0; t < TABLE_NUM; t++) {   /* shard_user.c:70-75 */
    tables[t] = calloc(1, sizeof(struct kvs));
    kvs_init(tables[t], hash_size[t]);
  }
  populate(pop);
  if (warm) warmup(pop, shard, G);
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
  if (nd == 5) dump(dumps);
  return 0;
}
