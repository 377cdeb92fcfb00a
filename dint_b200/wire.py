"""Wire formats and packet-type enums of the six reference servers, as numpy structured dtypes.

Each dtype is the reference's `#pragma pack(1) struct message`, byte for byte:
  lock_2pl/udp/net.h:11-31, lock_fasst/udp/net.h:11-31, log_server/udp/net.h:15-30,
  store/udp/net.h:15-41, tatp/udp/net.h:15-65, smallbank/udp/net.h:15-52.
"""
import numpy as np

LOCK2PL, FASST, LOG, STORE, TATP, SMALLBANK = range(6)
KIND_NAMES = ["lock_2pl", "lock_fasst", "log_server", "store", "tatp", "smallbank"]

MSG_DTYPE = [
    np.dtype([("action", "u1"), ("lid", "<u4"), ("type", "u1")]),
    np.dtype([("type", "u1"), ("lid", "<u4"), ("ver", "<u4")]),
    np.dtype([("type", "u1"), ("key", "<u8"), ("val", "u1", (40,)), ("ver", "<u4")]),
    np.dtype([("type", "u1"), ("key", "<u8"), ("val", "u1", (40,)), ("ver", "<u4")]),
    np.dtype([("ord", "u1"), ("type", "u1"), ("table", "u1"), ("key", "<u8"), ("val", "u1", (40,)), ("ver", "<u4")]),
    np.dtype([("ord", "u1"), ("type", "u1"), ("table", "u1"), ("key", "<u8"), ("val", "u1", (8,)), ("ver", "<u4")]),
]
MSG_SIZE = [d.itemsize for d in MSG_DTYPE]
assert MSG_SIZE == [6, 9, 53, 53, 55, 23]

# reference struct log_entry layouts (NOT packed): log_server/udp/utils.h:19-23, tatp/udp/kvs.h:23-29,
# smallbank/udp/kvs.h:20-25
LOG_ENTRY_SIZE = [0, 0, 56, 0, 64, 32]


class Lock2pl:            # lock_2pl/udp/net.h:11-23
    kAcquireLock, kReleaseLock, kGrantLock, kRejectLock, kRetry, kReleaseAck = range(6)
    kShared, kExclusive = 0, 1


class Fasst:              # lock_fasst/udp/net.h:11-21
    kRead, kAcquireLock, kAbort, kCommit, kGrantRead, kGrantLock, kRejectLock, kAbortAck, kCommitAck = range(9)


class Log:                # log_server/udp/net.h:15-18
    kCommit, kAck = 0, 1


class Store:              # store/udp/net.h:15-29
    kRead, kSet, kInsert, kGrantRead, kRejectRead, kSetAck, kRejectSet, kNotExist, kInsertAck, kRejectInsert = range(10)


class StoreEbpf:          # store/ebpf/utils.h:21-32: the eBPF store server's packet types (the same values)
    READ, SET, INSERT, GRANT_READ, REJECT_READ, SET_ACK, REJECT_SET, NOT_EXIST, INSERT_ACK, REJECT_INSERT = range(10)


class Tatp:               # tatp/udp/net.h:15-52
    (kRead, kAcquireLock, kAbort, kCommit, kGrantRead, kRejectRead, kNotExist, kGrantLock, kRejectLock,
     kAbortAck, kCommitAck, kRejectCommit, kCommitPrim, kCommitBck, kCommitLog, kCommitPrimAck,
     kCommitBckAck, kCommitLogAck, kInsertPrim, kInsertBck, kInsertPrimAck, kInsertBckAck, kDeletePrim,
     kDeleteBck, kDeleteLog, kDeletePrimAck, kDeleteBckAck, kDeleteLogAck) = range(28)
    # reply of the eBPF lock server (tatp/ebpf/utils.h:73, tatp/caladan/proto.h:52): the refused lock is held for the
    # same key; kRejectLock then means false sharing.  Sent only by engines created with lock_holder_keys.
    kRejectLockSameKey = 28
    kSubscriber, kSecondSubscriber, kAccessInfo, kSpecialFacility, kCallForwarding = range(5)


class TatpEbpf:           # tatp/ebpf/utils.h:40-73: the eBPF TATP shard server's packet types (the same values)
    (READ, ACQUIRE_LOCK, ABORT, COMMIT, GRANT_READ, REJECT_READ, NOT_EXIST, GRANT_LOCK, REJECT_LOCK, ABORT_ACK,
     COMMIT_ACK, REJECT_COMMIT, COMMIT_PRIM, COMMIT_BCK, COMMIT_LOG, COMMIT_PRIM_ACK, COMMIT_BCK_ACK, COMMIT_LOG_ACK,
     INSERT_PRIM, INSERT_BCK, INSERT_PRIM_ACK, INSERT_BCK_ACK, DELETE_PRIM, DELETE_BCK, DELETE_LOG, DELETE_PRIM_ACK,
     DELETE_BCK_ACK, DELETE_LOG_ACK, REJECT_LOCK_SAME_KEY) = range(29)


class Smallbank:          # smallbank/udp/net.h:15-38
    (kAcquireShared, kAcquireExclusive, kReleaseShared, kReleaseExclusive, kCommitPrim, kCommitBck,
     kCommitLog, kGrantShared, kRejectShared, kGrantExclusive, kRejectExclusive, kReleaseSharedAck,
     kReleaseExclusiveAck, kCommitPrimAck, kCommitBckAck, kCommitLogAck, kRetry, kWarmupRead,
     kWarmupReadAck) = range(19)
    kSaving, kChecking = 0, 1


class SmallbankEbpf:      # smallbank/ebpf/utils.h:31-50: the eBPF SmallBank shard server's packet types (the same values)
    (ACQUIRE_SHARED, ACQUIRE_EXCLUSIVE, RELEASE_SHARED, RELEASE_EXCLUSIVE, COMMIT_PRIM, COMMIT_BCK, COMMIT_LOG,
     GRANT_SHARED, REJECT_SHARED, GRANT_EXCLUSIVE, REJECT_EXCLUSIVE, RELEASE_SHARED_ACK, RELEASE_EXCLUSIVE_ACK,
     COMMIT_PRIM_ACK, COMMIT_BCK_ACK, COMMIT_LOG_ACK, RETRY, WARMUP_READ, WARMUP_READ_ACK) = range(19)
    SAVING, CHECKING = 0, 1


def as_records(kind, raw):
    """View a uint8 buffer of n*msg bytes as the structured wire dtype."""
    a = np.ascontiguousarray(raw, dtype=np.uint8).reshape(-1)
    return a.view(MSG_DTYPE[kind])


def as_bytes(rec):
    """View structured wire records as a flat uint8 array."""
    return np.ascontiguousarray(rec).view(np.uint8).reshape(-1)
