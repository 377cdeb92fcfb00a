# oracle/smallbank_ebpf.mk -- TEST INFRASTRUCTURE.  Builds _ref/smallbank_ebpf: the reference's eBPF SmallBank shard
# server -- its XDP and TC programs (smallbank/ebpf/shard_kern.c) and its table (smallbank/ebpf/kvs.h, populated as
# smallbank.h does), compiled UNMODIFIED where they lie under $(REF) as user-space C against the bpf_helpers.h stand-in
# in ebpf_shim/ -- driven one request at a time by smallbank_ebpf_replay.c.  Nothing is built when the reference
# sources are absent.
REF ?= /root/reference
CC ?= gcc
OUT = _ref
EBPF = $(REF)/smallbank/ebpf
EBPF_CFLAGS = -O2 -std=gnu11 -w -Iebpf_shim -I$(EBPF)
BINS = $(OUT)/smallbank_ebpf

all: $(if $(wildcard $(EBPF)/shard_kern.c),$(BINS),)

$(OUT)/smallbank_ebpf: smallbank_ebpf_replay.c $(EBPF)/shard_kern.c $(EBPF)/kvs.h $(EBPF)/smallbank.h ebpf_shim/linux/tools/lib/bpf/bpf_helpers.h
	@mkdir -p $(OUT)
	$(CC) $(EBPF_CFLAGS) -o $@ smallbank_ebpf_replay.c $(EBPF)/shard_kern.c

.PHONY: all
