# oracle/tatp_ebpf.mk -- TEST INFRASTRUCTURE.  Builds _ref/tatp_ebpf_shard and _ref/tatp_ebpf_lock: the reference's eBPF
# TATP shard server -- its XDP and TC programs (tatp/ebpf/shard_kern.c, and lock_kern.c, which adds a holder key beside
# every lock word) and its chained table (tatp/ebpf/kvs.h), compiled UNMODIFIED where they lie under $(REF) as
# user-space C against the bpf_helpers.h stand-in in ebpf_shim/ -- driven one request at a time by tatp_ebpf_replay.c.
# Nothing is built when the reference sources are absent.
REF ?= /root/reference
CC ?= gcc
OUT = _ref
EBPF = $(REF)/tatp/ebpf
EBPF_CFLAGS = -O2 -std=gnu11 -w -Iebpf_shim -I$(EBPF)
BINS = $(OUT)/tatp_ebpf_shard $(OUT)/tatp_ebpf_lock

all: $(if $(wildcard $(EBPF)/shard_kern.c),$(BINS),)

$(OUT)/tatp_ebpf_shard: tatp_ebpf_replay.c $(EBPF)/shard_kern.c $(EBPF)/kvs.h ebpf_shim/linux/tools/lib/bpf/bpf_helpers.h
	@mkdir -p $(OUT)
	$(CC) $(EBPF_CFLAGS) -o $@ tatp_ebpf_replay.c $(EBPF)/shard_kern.c
$(OUT)/tatp_ebpf_lock: tatp_ebpf_replay.c $(EBPF)/lock_kern.c $(EBPF)/kvs.h ebpf_shim/linux/tools/lib/bpf/bpf_helpers.h
	@mkdir -p $(OUT)
	$(CC) $(EBPF_CFLAGS) -DTATP_EBPF_LOCK=1 -o $@ tatp_ebpf_replay.c $(EBPF)/lock_kern.c

.PHONY: all
