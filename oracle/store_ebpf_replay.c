/* oracle/store_ebpf_replay.c -- TEST INFRASTRUCTURE.  Replays a trace through the reference's eBPF store server, built
 * from its unmodified sources (oracle/store_ebpf.mk links one of store/ebpf/store{,_wb,_wt}_kern.c, compiled as
 * user-space C against oracle/ebpf_shim, and includes store/ebpf/kvs.h).  One request at a time, as one server thread:
 *   XDP (tps_prim_xdp_main) -> XDP_TX: the reply leaves as it is;
 *                           -> XDP_PASS: the user-space dispatch below (the 3 branches of store_user.c:133-164;
 *                              store_wt_user.c drops the kvs_set_evict calls), then TC egress (tps_prim_tc_main)
 *                              on the reply, which is shrunk back to struct message.
 * A request of another type passes XDP untouched and store_user.c:164 panics: its reply is written as type 0xFF.
 *
 * usage: store_ebpf_<variant> REQ RESP [KEYS SETS TABLE] [--populate S]
 *   REQ / RESP: n packed 53-byte struct message; --populate S first serves the eBPF client's kInsert stream for S
 *   subscribers (store/caladan/client_ebpf.cc:137-180, 600 populate threads in thread order, bytes it leaves
 *   uninitialised are zero).  KEYS: u64 keys whose state is dumped: SETS gets the 232-byte struct cache_entry of each
 *   key's bucket, TABLE gets {u32 found, u32 ver, u8 val[40]} per key (kvs_get).  Prints "kv_count N" (valid table
 *   slots). */
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

#ifndef STORE_EBPF_WT
#define STORE_EBPF_WT 0
#endif

/* ---- bpf_map_lookup_elem of the shim: one lazily allocated zeroed array per map --------------------------------- */
static struct { const void *map; uint8_t *base; size_t vsz, n; } maps[8];
void *shim_map_lookup(const void *map, size_t value_size, size_t max_entries, uint32_t key) {
  int i = 0;
  for (; i < 8 && maps[i].map && maps[i].map != map; i++) {}
  if (i == 8) { fprintf(stderr, "too many maps\n"); exit(2); }
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
static struct cache_entry *cache_of(uint64_t key) {   /* the one array map of value struct cache_entry */
  for (int i = 0; i < 8 && maps[i].map; i++)
    if (maps[i].vsz == sizeof(struct cache_entry)) return (struct cache_entry *)maps[i].base + fasthash64(&key, 8, 0xdeadbeef) % KVS_HASH_SIZE;
  return NULL;
}

static struct kvs table;
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

/* one request in, one 53-byte reply out */
static void serve(const struct message *req, struct message *reply) {
  headers(40000, FASST_PORT, sizeof(struct message));
  memset(pkt + HDR, 0, sizeof(struct ext_message));
  memcpy(pkt + HDR, req, sizeof *req);
  struct xdp_md ctx;
  memset(&ctx, 0, sizeof ctx);
  ctx.data = (uint32_t)(uintptr_t)pkt;
  ctx.data_end = ctx.data + HDR + sizeof(struct message);
  if (tps_prim_xdp_main(&ctx) == XDP_TX) { memcpy(reply, pkt + HDR, sizeof *reply); return; }
  size_t got = ctx.data_end - ctx.data - HDR;
  struct ext_message msg;
  memset(&msg, 0, sizeof msg);
  memcpy(&msg, pkt + HDR, got < sizeof msg ? got : sizeof msg);
  if (got != sizeof msg || (msg.type != READ && msg.type != SET && msg.type != INSERT)) {   /* store_user.c:134,145,156,164 */
    memcpy(reply, req, sizeof *reply);
    reply->type = 0xFF;
    return;
  }
  /* ---- store_user.c:133-162 ---- */
  if (msg.type == READ) {
    if (!STORE_EBPF_WT && msg.ver1 == 1) kvs_set_evict(&table, msg.key2, msg.val2, msg.ver2);
    int res = kvs_get(&table, msg.key1, msg.val1, &msg.ver1);
    if (res == 0) msg.type = GRANT_READ;
    else msg.type = NOT_EXIST;
  } else if (msg.type == SET) {
    if (!STORE_EBPF_WT && msg.ver1 == 1) kvs_set_evict(&table, msg.key2, msg.val2, msg.ver2);
    kvs_set(&table, msg.key1, msg.val1, &msg.ver1);
    if (msg.ver1 != 0) msg.type = SET_ACK;
    else msg.type = NOT_EXIST;
  } else {
    kvs_insert(&table, msg.key1, msg.val1);
    if (!STORE_EBPF_WT) kvs_set_evict(&table, msg.key2, msg.val2, msg.ver2);
    msg.type = INSERT_ACK;
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

static void populate(uint32_t S) {   /* store/caladan/client_ebpf.cc:137-180 with threads = 600 (:282) */
  const uint32_t threads = 600, slice = S / threads;
  struct message msg, reply;
  memset(&msg, 0, sizeof msg);
  for (uint32_t w = 0; w < threads; w++) {
    uint64_t seed = 0xdeadbeef;
    uint32_t lo = w * slice, hi = (w == threads - 1) ? S : (w + 1) * slice;
    for (uint32_t s = lo; s < hi; s++)
      for (uint64_t sf = 1; sf <= 4; sf++)
        for (uint64_t st = 0; st <= 16; st += 8) {
          uint8_t val[VAL_SIZE] = {0};
          val[1] = 0x5a;                                       /* numberx[0] = kValMagic */
          seed = seed * 1103515245 + 12345;                    /* fastrand, store/caladan/tatp.h:37-40 */
          val[0] = (uint8_t)((uint32_t)(seed >> 32) % 24 + 1); /* end_time */
          msg.key = (uint64_t)s | (sf << 32) | (st << 40);
          memcpy(msg.val, val, VAL_SIZE);
          msg.type = INSERT;
          serve(&msg, &reply);
          msg = reply;                                         /* the client reuses the buffer the reply landed in */
        }
  }
}

int main(int argc, char **argv) {
  uint32_t pop = 0;
  const char *pos[5] = {0};
  int np = 0;
  for (int i = 1; i < argc; i++) {
    if (!strcmp(argv[i], "--populate") && i + 1 < argc) pop = (uint32_t)strtoul(argv[++i], NULL, 0);
    else if (np < 5) pos[np++] = argv[i];
  }
  if (np != 2 && np != 5) {
    fprintf(stderr, "usage: %s REQ RESP [KEYS SETS TABLE] [--populate S]\n", argv[0]);
    return 2;
  }
  pkt = mmap(NULL, 4096, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_32BIT, -1, 0);
  if (pkt == MAP_FAILED) { perror("mmap"); return 2; }
  kvs_init(&table, KVS_HASH_SIZE);
  if (pop) populate(pop);
  size_t len = 0;
  struct message *req = slurp(pos[0], &len);
  size_t n = len / sizeof(struct message);
  FILE *out = wopen(pos[1]);
  for (size_t i = 0; i < n; i++) {
    struct message reply;
    serve(&req[i], &reply);
    fwrite(&reply, sizeof reply, 1, out);
  }
  fclose(out);
  if (np == 5) {
    uint64_t *keys = slurp(pos[2], &len);
    size_t nk = len / 8;
    FILE *fs = wopen(pos[3]), *ft = wopen(pos[4]);
    for (size_t i = 0; i < nk; i++) {
      static const struct cache_entry none;   /* no request reached XDP: the map was never allocated */
      const struct cache_entry *ce = cache_of(keys[i]);
      fwrite(ce ? ce : &none, sizeof(struct cache_entry), 1, fs);
      struct { uint32_t found, ver; uint8_t val[VAL_SIZE]; } t;
      memset(&t, 0, sizeof t);
      t.found = kvs_get(&table, keys[i], t.val, &t.ver) == 0;
      fwrite(&t, sizeof t, 1, ft);
    }
    fclose(fs);
    fclose(ft);
  }
  uint64_t count = 0;
  for (int b = 0; b < table.hash_size; b++)
    for (struct kvs_entry *e = table.bucket_heads[b]; e; e = e->next)
      for (int j = 0; j < KEYS_PER_ENTRY; j++) count += e->valid[j] != 0;
  printf("kv_count %llu\n", (unsigned long long)count);
  return 0;
}
