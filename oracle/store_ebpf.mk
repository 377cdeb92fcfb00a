# oracle/store_ebpf.mk -- TEST INFRASTRUCTURE.  Builds _ref/store_ebpf_{wb_bloom,wb,wt}: the reference's eBPF store
# server -- its XDP and TC programs (store/ebpf/store{,_wb,_wt}_kern.c) and its table (store/ebpf/kvs.h), compiled
# UNMODIFIED where they lie under $(REF) as user-space C against the bpf_helpers.h stand-in in ebpf_shim/ -- driven one
# request at a time by store_ebpf_replay.c.  Nothing is built when the reference sources are absent.
REF ?= /root/reference
CC ?= gcc
OUT = _ref
EBPF = $(REF)/store/ebpf
EBPF_CFLAGS = -O2 -std=gnu11 -w -Iebpf_shim -I$(EBPF)
BINS = $(OUT)/store_ebpf_wb_bloom $(OUT)/store_ebpf_wb $(OUT)/store_ebpf_wt

all: $(if $(wildcard $(EBPF)/store_kern.c),$(BINS),)

$(OUT)/store_ebpf_wb_bloom: store_ebpf_replay.c $(EBPF)/store_kern.c ebpf_shim/linux/tools/lib/bpf/bpf_helpers.h
	@mkdir -p $(OUT)
	$(CC) $(EBPF_CFLAGS) -o $@ store_ebpf_replay.c $(EBPF)/store_kern.c
$(OUT)/store_ebpf_wb: store_ebpf_replay.c $(EBPF)/store_wb_kern.c ebpf_shim/linux/tools/lib/bpf/bpf_helpers.h
	@mkdir -p $(OUT)
	$(CC) $(EBPF_CFLAGS) -o $@ store_ebpf_replay.c $(EBPF)/store_wb_kern.c
$(OUT)/store_ebpf_wt: store_ebpf_replay.c $(EBPF)/store_wt_kern.c ebpf_shim/linux/tools/lib/bpf/bpf_helpers.h
	@mkdir -p $(OUT)
	$(CC) $(EBPF_CFLAGS) -DSTORE_EBPF_WT=1 -o $@ store_ebpf_replay.c $(EBPF)/store_wt_kern.c

.PHONY: all
