"""Key-space sharding over the GPUs of one box: one process per GPU (torchrun), torch.distributed for the
plumbing (NCCL on GPUs, gloo in the CPU tests).

The reference shards on the CLIENT (key % 3, tatp/caladan/client_udp_shard.cc:187) and its servers never
talk to each other.  Here every rank receives an arbitrary slice of the request stream, and the engine
routes each request to the shard that owns its lock slot / bucket (SURVEY.md section 8(e)):

    owner      = slot % world                       slot = fasthash64(key) % table_size, exactly the slot
                                                    ONE reference server would use, so collisions are unchanged
    dispatch   = stable partition by owner -> all-to-all (variable counts) of fixed-size wire records
    local step = the shard's Engine (n_shards = world, shard_id = rank) on what it received
    combine    = all-to-all back -> inverse permutation

Order rule for bit-exactness: the global request order is rank-major (rank 0's slice first); a stable
partition keeps that order inside every destination, and all_to_all concatenates sources in rank order,
so each shard sees its requests in global order.  The result equals ONE sequential server processing
the concatenation of all ranks' slices.
"""
import ctypes as C
import os

import numpy as np
import torch
import torch.distributed as dist

from . import wire
from .engine import Engine, default_cfg, lib, DintPeerPtrs, DintError


def group_moduli(kind, cfg):
    """Group modulus per table, as the engine derives it (kv.cuh kv_create_tables)."""
    S, A = cfg.subs_sizing, cfg.accts_sizing
    if kind in (wire.LOCK2PL, wire.FASST):
        return [cfg.lock_slots, 1, 1, 1, 1]
    if kind == wire.STORE:
        return [S * 18 // 4, 1, 1, 1, 1]
    if kind == wire.TATP:
        return [4 * (S * 3 // 2 // 4), 4 * (S * 3 // 2 // 4), 4 * (S * 15 // 4 // 4), 4 * (S * 15 // 4 // 4), 4 * (S * 45 // 8 // 4)]
    if kind == wire.SMALLBANK:
        return [4 * (A * 3 // 2 // 4)] * 2 + [1, 1, 1]
    return [1] * 5


def owners_cpu(kind, cfg, world, rank, req):
    """Host twin of Engine.route_owner (libdint_wl.so), for the gloo tests."""
    from .workloads import lib as wl_lib
    L = wl_lib()
    L.dint_wl_owner.argtypes = [C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
    L.dint_wl_owner.restype = None
    mods = (C.c_uint32 * 5)(*group_moduli(kind, cfg))
    raw = np.ascontiguousarray(req, dtype=np.uint8).reshape(-1)
    n = raw.size // wire.MSG_SIZE[kind]
    out = np.empty(n, dtype=np.uint8)
    L.dint_wl_owner(kind, mods, world, rank, raw.ctypes.data, n, out.ctypes.data)
    return out


class ShardedEngine:
    """Collective engine: every rank calls submit*() with its slice of the request stream.

    local_submit (optional) replaces the GPU engine by any callable req_bytes -> resp_bytes (the CPU tests
    plug the oracle in to check the routing logic without a GPU)."""

    def __init__(self, kind, device=None, local_submit=None, group=None, by_dst=False, use_slabs=False, strict=True,
                 slab_slack=None, use_p2p=False, p2p_max_n=1 << 20, **cfg_over):
        """by_dst=True: tatp / smallbank placement -- the CLIENT names the destination shard of every record
        (primary key % G, backups, log); each rank is one complete `server_shard` (n_shards = 1) that
        populates only the keys it is a replica holder of (cfg txn_shards = world)."""
        self.kind = kind
        self.msg = wire.MSG_SIZE[kind]
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.cfg = default_cfg(kind, **cfg_over) if local_submit is None else None
        self._cfg_over = cfg_over
        self.local_submit = local_submit
        self.engine = None
        if local_submit is None:
            self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
            if by_dst:
                self.engine = Engine(kind, device=self.device.index, txn_shards=self.world, txn_shard_id=self.rank, **cfg_over)
            else:
                self.engine = Engine(kind, device=self.device.index, n_shards=self.world, shard_id=self.rank, **cfg_over)
        else:
            self.device = torch.device("cpu")
            from . import engine as _e
            self.cfg = _e.DintCfg()
            # only the sizing fields matter for routing
            self.cfg.lock_slots = cfg_over.get("lock_slots", 36000000)
            self.cfg.subs_sizing = cfg_over.get("subs_sizing", 7000000 if kind == wire.TATP else 2000000)
            self.cfg.accts_sizing = cfg_over.get("accts_sizing", 24000000)
        self.use_slabs, self.strict = use_slabs, strict
        self.slab_slack = slab_slack if slab_slack is not None else (1.5 if by_dst else 1.02)
        self.overflow = torch.zeros(2, dtype=torch.int32, device=self.device) if self.engine is not None else None
        self.use_p2p = False
        if use_p2p and self.engine is not None:
            self._init_p2p(p2p_max_n)

    # ---- fused dispatch / combine over NVLink peer memory -------------------------------------------
    def _cap(self, n):
        mean = (n + self.world - 1) // self.world
        cap = int(mean * self.slab_slack) + int(8 * (mean ** 0.5)) + 64
        return (cap + 127) // 128 * 128          # whole engine tiles: a reply tile never straddles two sources' slabs

    def _init_p2p(self, max_n, n_sets=3):
        """Symmetric buffer per rank: n_sets x {inbox [world][cap] | return buffer [world][cap]} | signal block, mapped by
        all peers (torch symmetric memory = CUDA IPC + peer access over NVLink); the step itself is driven by the
        library (dint_shard_submit_many)."""
        import torch.distributed._symmetric_memory as symm_mem
        W = self.world
        self.p2p_max_n = max_n
        cap = self._cap(max_n)
        region = (W * cap * self.msg + 255) // 256 * 256
        k = 2                                                    # regions per set: inbox | return buffer
        self.sym = symm_mem.empty(n_sets * k * region + 4096, dtype=torch.uint8, device=self.device)
        grp = self.group if self.group is not None else dist.group.WORLD
        self.sym_hdl = symm_mem.rendezvous(self.sym, group=grp.group_name)
        self.sym.zero_()
        torch.cuda.synchronize(self.device)
        self.sym_hdl.barrier()
        ptrs = [int(p) for p in self.sym_hdl.buffer_ptrs]
        inbox = (DintPeerPtrs * n_sets)(*[DintPeerPtrs.of([p + s * k * region for p in ptrs]) for s in range(n_sets)])
        retbox = (DintPeerPtrs * n_sets)(*[DintPeerPtrs.of([p + s * k * region + region for p in ptrs]) for s in range(n_sets)])
        sig = DintPeerPtrs.of([p + n_sets * k * region for p in ptrs])
        ctx = C.c_void_p()
        rc = lib().dint_shard_create(self.engine.h, W, self.rank, cap, n_sets, inbox, retbox, C.byref(sig), max_n, C.byref(ctx))
        if rc != 0:
            raise DintError(rc, "dint_shard_create")
        self.p2p_ctx = ctx
        self.use_p2p = True

    def _p2p_many(self, reqs, dsts=None, caps=None):
        """k batches through dint_shard_submit_many_v (the same k on every rank; sizes may differ).  caps: per batch the
        slab capacity to use (the same on every rank; see cap_for) -- None = the full capacity."""
        k = len(reqs)
        ns = [r.numel() // self.msg for r in reqs]
        assert all(r.is_contiguous() for r in reqs) and all(0 < n <= self.p2p_max_n for n in ns)
        outs = [torch.empty(n * self.msg, dtype=torch.uint8, device=self.device) for n in ns]
        a_req = (C.c_void_p * k)(*[r.data_ptr() for r in reqs])
        a_out = (C.c_void_p * k)(*[o.data_ptr() for o in outs])
        a_dst = None if dsts is None or dsts[0] is None else (C.c_void_p * k)(*[d.data_ptr() for d in dsts])
        s = torch.cuda.current_stream(self.device).cuda_stream
        if caps is None and all(n == ns[0] for n in ns):      # equally sized batches at the full slab capacity
            rc = lib().dint_shard_submit_many(self.p2p_ctx, k, a_req, a_dst, ns[0], a_out, C.c_void_p(s) if s else None)
            if rc != 0:
                raise DintError(rc, "dint_shard_submit_many")
            return outs
        a_n = (C.c_uint64 * k)(*ns)
        a_cap = None if caps is None else (C.c_uint32 * k)(*caps)
        rc = lib().dint_shard_submit_many_v(self.p2p_ctx, k, a_req, a_dst, a_n, a_cap, a_out, C.c_void_p(s) if s else None)
        if rc != 0:
            raise DintError(rc, "dint_shard_submit_many_v")
        return outs

    def cap_for(self, n_max):
        """Slab capacity for a batch whose LARGEST per-rank size is n_max (every rank must pass the same value)."""
        return min(self._cap(n_max), self._cap(self.p2p_max_n))

    def submit_many_host(self, reqs, outs, dsts=None):
        """k equally sized batches from / to pinned HOST tensors through dint_shard_submit_host (H2D | dispatch | engine |
        combine | D2H pipelined inside the library); returns when every out is complete."""
        k = len(reqs)
        n = reqs[0].numel() // self.msg
        a_req = (C.c_void_p * k)(*[r.data_ptr() for r in reqs])
        a_out = (C.c_void_p * k)(*[o.data_ptr() for o in outs])
        a_dst = None if dsts is None or dsts[0] is None else (C.c_void_p * k)(*[d.data_ptr() for d in dsts])
        rc = lib().dint_shard_submit_host(self.p2p_ctx, k, a_req, a_dst, n, a_out)
        if rc != 0:
            raise DintError(rc, "dint_shard_submit_host")
        return outs

    def _submit_gpu_p2p(self, req, n, dst):
        """Dispatch partitions the batch and stores every run straight into the owners' inboxes (then raises their epoch
        flags); the owners' apply kernel stores the replies straight into this rank's return buffer; combine reassembles
        them locally.  No NCCL call, no host round trip."""
        return self._p2p_many([req], [dst])[0]

    def check_p2p(self):
        """(overflowed records, timed-out waits) since the last check; both must be 0 for the results to stand."""
        v = (C.c_uint32 * 2)()
        rc = lib().dint_shard_flags(self.p2p_ctx, v)
        if rc != 0:
            raise DintError(rc, "dint_shard_flags")
        return int(v[0]), int(v[1])

    def close(self):
        if self.use_p2p:
            lib().dint_shard_destroy(self.p2p_ctx)
            self.use_p2p = False
        if self.engine is not None:
            self.engine.close()
            self.engine = None

    def populate(self):
        self.engine.populate()       # dint_load keeps only this shard's keys

    # ---- the collective request path -------------------------------------------------------------
    def submit_tensor(self, req, dst=None):
        """req: uint8 tensor [n * msg] on this rank's device; returns the replies, same layout/order.
        dst: optional uint8 tensor [n] of client-chosen destination shards (tatp / smallbank)."""
        n = req.numel() // self.msg
        if self.engine is not None:
            return self._submit_gpu(req, n, dst)
        rec = req.view(n, self.msg)
        owner = dst if dst is not None else torch.from_numpy(owners_cpu(self.kind, self.cfg, self.world, self.rank, req.numpy()))
        # dispatch: stable partition by owner
        order = torch.argsort(owner, stable=True)
        send_counts = torch.bincount(owner.long(), minlength=self.world)[: self.world]
        recv_counts = torch.empty_like(send_counts)
        dist.all_to_all_single(recv_counts, send_counts, group=self.group)
        sc, rc = send_counts.tolist(), recv_counts.tolist()
        send = rec.index_select(0, order).contiguous()
        m = int(sum(rc))
        recv = torch.empty((m, self.msg), dtype=torch.uint8)
        dist.all_to_all_single(recv, send, output_split_sizes=rc, input_split_sizes=sc, group=self.group)
        out_local = torch.from_numpy(np.asarray(self.local_submit(recv.numpy().reshape(-1)))).view(m, self.msg) if m else recv
        back = torch.empty((n, self.msg), dtype=torch.uint8)
        dist.all_to_all_single(back, out_local.contiguous(), output_split_sizes=sc, input_split_sizes=rc, group=self.group)
        out = torch.empty_like(rec)
        out.index_copy_(0, order, back)
        return out.view(-1)

    def _dispatch_local(self, req, n, dst):
        """Partition into a local send buffer of `world` slabs; returns (slabs, state, cap)."""
        eng, W = self.engine, self.world
        cap = self._cap(n)
        slabs = torch.empty(W * cap * self.msg, dtype=torch.uint8, device=req.device)
        ptrs = Engine.slab_ptrs(slabs.data_ptr(), W, cap * self.msg)
        state = eng.route_dispatch(req, n, W, self.rank, cap, ptrs, self.overflow, owner_in=dst)
        return slabs, state, cap

    def _submit_gpu_slabs(self, req, n, dst):
        """Fixed-capacity exchange: every rank sends every peer one slab of `cap` records (real ones first, the
        rest padding), so the all-to-all needs no split sizes from the device -- no host round trip inside the
        step.  The local engine runs ONE batch of world * cap records in source-rank order; padding records are
        answered unchanged.  A slab overflow (counted on the device) means the result must be discarded."""
        eng, W = self.engine, self.world
        slabs, state, cap = self._dispatch_local(req, n, dst)
        recv = torch.empty_like(slabs)
        dist.all_to_all_single(recv, slabs, group=self.group)
        out_local = torch.empty_like(recv)
        eng.submit_tensor(recv, out_local)
        back = torch.empty_like(slabs)
        dist.all_to_all_single(back, out_local, group=self.group)
        out = torch.empty(n * self.msg, dtype=torch.uint8, device=req.device)
        return eng.route_combine(Engine.slab_ptrs(back.data_ptr(), W, cap * self.msg), state, n, W, cap, out)

    def submit_many(self, reqs, dsts=None, caps=None):
        """A sequence of collective batches (each rank passes equally many, equally sized tensors), software
        pipelined: batch k+1 is partitioned and exchanged on a side stream while batch k runs through the
        local engine and its replies travel back on the main stream.  The engine still sees the batches in
        order, so the result equals calling submit_tensor() on each batch in turn."""
        eng, W = self.engine, self.world
        if self.use_p2p and reqs[0].numel() // self.msg <= self.p2p_max_n:
            return self._p2p_many(reqs, dsts, caps)
        assert dsts is None, "client-chosen shards: use the p2p step or submit_tensor"
        main = torch.cuda.current_stream(self.device)
        if not hasattr(self, "_side"):
            self._side = torch.cuda.Stream(self.device)
        side = self._side
        side.wait_stream(main)
        keep = []

        def dispatch(req):
            n = req.numel() // self.msg
            cap = self._cap(n)
            with torch.cuda.stream(side):
                slabs, state, _ = self._dispatch_local(req, n, None)
                recv = torch.empty_like(slabs)
                dist.all_to_all_single(recv, slabs, group=self.group)
                ev = torch.cuda.Event()
                ev.record(side)
            keep.extend([slabs, state, recv])
            return recv, (state, cap), ev, n

        if not hasattr(self, "_ret"):
            self._ret = torch.cuda.Stream(self.device)
        ret = self._ret
        ret.wait_stream(main)
        outs = []
        nxt = dispatch(reqs[0])
        for k in range(len(reqs)):
            recv, perm, ev, n = nxt
            if k + 1 < len(reqs):
                nxt = dispatch(reqs[k + 1])
            main.wait_event(ev)
            out_local = torch.empty_like(recv)
            eng.submit_tensor(recv, out_local)               # main stream: the engine sees the batches in order
            done = torch.cuda.Event()
            done.record(main)
            with torch.cuda.stream(ret):                     # replies travel back while the next batch computes
                ret.wait_event(done)
                back = torch.empty_like(recv)
                dist.all_to_all_single(back, out_local, group=self.group)
                out = torch.empty(n * self.msg, dtype=torch.uint8, device=self.device)
                state, cap = perm
                outs.append(eng.route_combine(Engine.slab_ptrs(back.data_ptr(), W, cap * self.msg), state, n, W, cap, out))
            keep.extend([out_local, back])
        main.wait_stream(ret)
        main.wait_stream(side)
        self._keep = keep               # buffers of the side streams stay referenced until the next call
        return outs

    def check_overflow(self):
        """True if any fixed-capacity exchange since the last check dropped a record (results invalid)."""
        v = int(self.overflow[0].item())
        self.overflow.zero_()
        return v != 0

    def _submit_gpu(self, req, n, dst):
        if self.use_p2p and 0 < n <= self.p2p_max_n:
            out = self._submit_gpu_p2p(req, n, dst)
            if self.strict and self.check_p2p() != (0, 0):
                raise RuntimeError("p2p exchange overflowed a slab or timed out")
            return out
        if self.use_slabs and n >= self.world * 1024:
            out = self._submit_gpu_slabs(req, n, dst)
            if not self.strict:
                return out
            if not self.check_overflow():
                return out
            raise RuntimeError("slab overflow in a strict fixed-capacity exchange: state already advanced; use use_slabs=False "
                               "for adversarially skewed traffic")
        return self._submit_gpu_exact(req, n, dst)

    def _submit_gpu_exact(self, req, n, dst):
        """GPU path: dispatch / combine with the library's own kernels (k_route_owner, k_exact_count/scan/scatter,
        k_exact_unpermute); NCCL moves the partitioned wire records."""
        eng = self.engine
        owner = dst if dst is not None else eng.route_owner(req)
        send, perm, counts = eng.route_partition(req, owner, self.world)
        recv_counts = torch.empty_like(counts)
        dist.all_to_all_single(recv_counts, counts, group=self.group)
        both = torch.stack([counts, recv_counts]).cpu()                # the one host sync: split sizes
        sc, rc = both[0].tolist(), both[1].tolist()
        m = int(sum(rc))
        recv = torch.empty((m, self.msg), dtype=torch.uint8, device=req.device)
        dist.all_to_all_single(recv, send.view(n, self.msg), output_split_sizes=rc, input_split_sizes=sc, group=self.group)
        out_local = torch.empty_like(recv)
        if m:
            eng.submit_tensor(recv.view(-1), out_local.view(-1))
        back = torch.empty((n, self.msg), dtype=torch.uint8, device=req.device)
        dist.all_to_all_single(back, out_local, output_split_sizes=sc, input_split_sizes=rc, group=self.group)
        return eng.route_unpermute(back.view(-1), perm)

    def submit(self, req_host, dst_host=None):
        """Host path: numpy uint8 in, numpy uint8 out (H2D, collective device step, D2H)."""
        t = torch.from_numpy(np.ascontiguousarray(req_host, dtype=np.uint8).reshape(-1))
        d = None if dst_host is None else torch.from_numpy(np.ascontiguousarray(dst_host, dtype=np.uint8))
        if self.engine is not None:
            t = t.to(self.device, non_blocking=True)
            d = None if d is None else d.to(self.device, non_blocking=True)
        out = self.submit_tensor(t, d)
        return out.cpu().numpy()
