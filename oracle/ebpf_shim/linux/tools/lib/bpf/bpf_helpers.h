/* oracle/ebpf_shim -- TEST INFRASTRUCTURE.  Stands in for linux/tools/lib/bpf/bpf_helpers.h so that the reference's
 * eBPF store programs (store/ebpf/store*_kern.c) compile unmodified as user-space C (oracle/store_ebpf.mk).  Maps are
 * lazily allocated zeroed arrays; the two packet-resizing helpers move data_end.  Packet addresses live in __u32
 * fields of xdp_md / __sk_buff, so the replay driver maps its packet buffers below 4 GB (MAP_32BIT). */
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <arpa/inet.h>
#include <linux/bpf.h>
#include <linux/pkt_cls.h>

#define SEC(name)
#define __uint(name, val) int (*name)[val]
#define __type(name, val) typeof(val) *name

/* array map lookup: value array of max_entries elements, allocated (zeroed) on first use */
void *shim_map_lookup(const void *map, size_t value_size, size_t max_entries, uint32_t key);
#define bpf_map_lookup_elem(map, key) \
  shim_map_lookup((map), sizeof(*(map)->value), sizeof(*(map)->max_entries) / sizeof(int), *(const uint32_t *)(key))

static inline long bpf_xdp_adjust_tail(struct xdp_md *ctx, int delta) {
  ctx->data_end += (uint32_t)delta;
  return 0;
}
static inline long bpf_skb_change_tail(struct __sk_buff *skb, uint32_t len, uint64_t flags) {
  (void)flags;
  skb->len = len;
  skb->data_end = skb->data + len;
  return 0;
}
