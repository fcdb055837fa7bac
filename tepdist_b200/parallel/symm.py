"""Symmetric (peer-mapped) device memory for the fused NVLink kernels (ops/csrc/comm_sm90.cu).

Every rank allocates the same-sized buffer, exports a CUDA IPC handle, and maps all peers' buffers; kernels then
read / write peer memory directly over NVLink (P2P loads/stores), replacing NCCL for the hot collectives.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional

import torch
import torch.distributed as dist

from .. import ops


class _CudaArray:
    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}


def _sigs(lib):
    vp, i, ll, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float
    pp = ctypes.POINTER(ctypes.c_void_p)
    table = {
        "tepd_symm_alloc": [ll, pp], "tepd_symm_free": [vp], "tepd_ipc_get_handle": [vp, vp], "tepd_ipc_open": [vp, pp],
        "tepd_ipc_close": [vp], "tepd_ipc_handle_size": [],
        "tepd_symm_barrier": [pp, i, i, vp, vp],
        "tepd_fused_rs_adamw_ag": [pp, pp, vp, vp, vp, i, ll, ll, ll, f, f, f, f, vp, i, vp, i],
    }
    for k, a in table.items():
        fn = getattr(lib, k)
        fn.restype = ctypes.c_int
        fn.argtypes = a


_VMM_STATE: dict = {}


def _vmm_sigs(lib):
    vp, i, ll, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float
    ull = ctypes.c_ulonglong
    pi, pll, pull, pp = ctypes.POINTER(i), ctypes.POINTER(ll), ctypes.POINTER(ull), ctypes.POINTER(ctypes.c_void_p)
    table = {
        "tepd_vmm_query": [i, i, pi, pll], "tepd_vmm_create": [i, ll, pull, pi], "tepd_vmm_import_fd": [i, pull],
        "tepd_vmm_map": [ull, i, ll, ll, pp], "tepd_vmm_unmap": [vp, ll], "tepd_vmm_release": [ull],
        "tepd_mc_create": [i, ll, pull, pi], "tepd_mc_add_device": [ull, i], "tepd_mc_bind": [ull, ull, ll],
        "tepd_mc_barrier": [vp, vp, vp, i, vp, vp],
        "tepd_mc_all_reduce_bf16": [vp, vp, vp, vp, i, i, ll, i, vp, vp, vp, i, vp],
        "tepd_mc_rs_adamw_ag": [vp, vp, vp, vp, vp, ll, ll, ll, f, f, f, f, vp, i, i, vp],
    }
    for k, a in table.items():
        fn = getattr(lib, k)
        fn.restype = ctypes.c_int
        fn.argtypes = a


def _exchange_fds(fds: List[int], group) -> dict:
    """Every rank hands `fds` (POSIX handles of its physical allocations) to every other rank of `group` over abstract
    AF_UNIX sockets with SCM_RIGHTS -- the way a file descriptor crosses a process boundary without ptrace rights.
    Returns {rank: [fd, ...]} with the receiver-side descriptor numbers (own entry = the fds passed in)."""
    import socket
    import struct
    import uuid
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    tok = [uuid.uuid4().hex if rank == 0 else None]
    dist.broadcast_object_list(tok, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    names = [f"\0tepd-{tok[0]}-{r}" for r in range(world)]
    srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    srv.bind(names[rank])
    srv.listen(world)
    dist.barrier(group)                       # everybody is listening
    for p in range(world):
        if p == rank:
            continue
        c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        c.connect(names[p])
        socket.send_fds(c, [struct.pack("i", rank)], list(fds))
        c.close()
    got = {rank: list(fds)}
    srv.settimeout(120)
    for _ in range(world - 1):
        conn, _a = srv.accept()
        msg, rfds, _f, _ad = socket.recv_fds(conn, 16, 8)
        got[struct.unpack("i", msg[:4])[0]] = list(rfds)
        conn.close()
    srv.close()
    dist.barrier(group)
    return got


def symm_backend(group=None) -> str:
    """'vmm' when every rank of the group can bind VMM allocations to an NVSwitch multicast object (NVLS), else 'ipc'
    (cudaIpc peer mappings, no multicast).  TEPDIST_SYMM=ipc|vmm overrides the probe."""
    import os
    forced = os.environ.get("TEPDIST_SYMM")
    if forced in ("ipc", "vmm"):
        return forced
    key = id(group) if group is not None else 0
    if key not in _VMM_STATE:
        lib = ops.lib()
        _vmm_sigs(lib)
        sup, gran = ctypes.c_int(0), ctypes.c_longlong(0)
        rc = lib.tepd_vmm_query(torch.cuda.current_device(), dist.get_world_size(group), ctypes.byref(sup), ctypes.byref(gran))
        mine = bool(rc == 0 and sup.value and gran.value > 0)
        everyone: List[Optional[bool]] = [None] * dist.get_world_size(group)
        dist.all_gather_object(everyone, mine, group=group)
        _VMM_STATE[key] = "vmm" if all(everyone) else "ipc"
    return _VMM_STATE[key]


class SymmetricBuffer:
    """nbytes of device memory on every rank of `group`, mutually mapped.

    backend 'vmm' (default on NVSwitch boxes): cuMemCreate physical pages, POSIX-fd handles exchanged over unix sockets,
    every peer's pages mapped into this process (`ptrs[r]`, unicast) AND all of them bound to one multicast object whose
    mapping `mc_ptr` addresses the n replicas at once: `multimem.ld_reduce` on it returns the switch-reduced value,
    `multimem.st` writes every replica (ops/csrc/vmm_sm90.cu).  backend 'ipc': cudaMalloc + cudaIpc handles, `mc_ptr` None."""

    def __init__(self, nbytes: int, group=None, backend: Optional[str] = None):
        self.lib = ops.lib()
        _sigs(self.lib)
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.backend = backend or symm_backend(group)
        self.mc_ptr: Optional[int] = None
        if self.backend == "vmm":
            self._init_vmm(nbytes)
        else:
            self._init_ipc(nbytes)
        self.ptr_array = (ctypes.c_void_p * self.world)(*self.ptrs)

    def _init_ipc(self, nbytes: int) -> None:
        self.nbytes = (nbytes + 255) // 256 * 256
        p = ctypes.c_void_p()
        rc = self.lib.tepd_symm_alloc(self.nbytes, ctypes.byref(p))
        if rc:
            raise RuntimeError(f"symmetric alloc failed ({rc})")
        self.local_ptr = p.value
        hs = self.lib.tepd_ipc_handle_size()
        h = ctypes.create_string_buffer(hs)
        rc = self.lib.tepd_ipc_get_handle(self.local_ptr, h)
        if rc:
            raise RuntimeError(f"cudaIpcGetMemHandle failed ({rc})")
        handles: List[Optional[bytes]] = [None] * self.world
        dist.all_gather_object(handles, bytes(h.raw), group=self.group)
        self.ptrs: List[int] = []
        for r, hb in enumerate(handles):
            if r == self.rank:
                self.ptrs.append(self.local_ptr)
                continue
            q = ctypes.c_void_p()
            rc = self.lib.tepd_ipc_open(ctypes.create_string_buffer(hb, hs), ctypes.byref(q))
            if rc:
                raise RuntimeError(f"cudaIpcOpenMemHandle(rank {r}) failed ({rc})")
            self.ptrs.append(q.value)

    def _init_vmm(self, nbytes: int) -> None:
        import os
        lib = self.lib
        _vmm_sigs(lib)
        dev = torch.cuda.current_device()
        sup, gran = ctypes.c_int(0), ctypes.c_longlong(0)
        rc = lib.tepd_vmm_query(dev, self.world, ctypes.byref(sup), ctypes.byref(gran))
        if rc or gran.value <= 0:
            raise RuntimeError(f"VMM API unavailable ({rc})")
        g = gran.value
        self.nbytes = (max(nbytes, 1) + g - 1) // g * g
        use_mc = bool(sup.value) and self.world > 1

        def chk(rc, what):
            if rc:
                raise RuntimeError(f"{what} failed ({rc}) on rank {self.rank}")

        mem, fd = ctypes.c_ulonglong(0), ctypes.c_int(-1)
        chk(lib.tepd_vmm_create(dev, self.nbytes, ctypes.byref(mem), ctypes.byref(fd)), "cuMemCreate/export")
        send = [fd.value]
        mc = ctypes.c_ulonglong(0)
        if use_mc and self.rank == 0:
            mfd = ctypes.c_int(-1)
            chk(lib.tepd_mc_create(self.world, self.nbytes, ctypes.byref(mc), ctypes.byref(mfd)), "cuMulticastCreate")
            send.append(mfd.value)
        got = _exchange_fds(send, self.group) if self.world > 1 else {self.rank: send}
        self.ptrs = []
        self._handles = []
        for r in range(self.world):
            h = mem
            if r != self.rank:
                h = ctypes.c_ulonglong(0)
                chk(lib.tepd_vmm_import_fd(got[r][0], ctypes.byref(h)), f"import of rank {r}'s allocation")
            q = ctypes.c_void_p()
            chk(lib.tepd_vmm_map(h.value, dev, self.nbytes, g, ctypes.byref(q)), f"map of rank {r}'s allocation")
            self.ptrs.append(q.value)
            self._handles.append(h.value)
        self.local_ptr = self.ptrs[self.rank]
        if use_mc:
            if self.rank != 0:
                chk(lib.tepd_vmm_import_fd(got[0][1], ctypes.byref(mc)), "import of the multicast object")
            chk(lib.tepd_mc_add_device(mc.value, dev), "cuMulticastAddDevice")
            dist.barrier(self.group)               # every device is part of the object before anybody binds memory
            chk(lib.tepd_mc_bind(mc.value, mem.value, self.nbytes), "cuMulticastBindMem")
            q = ctypes.c_void_p()
            chk(lib.tepd_vmm_map(mc.value, dev, self.nbytes, g, ctypes.byref(q)), "map of the multicast object")
            self.mc_ptr = q.value
            self._mc_handle = mc.value
            dist.barrier(self.group)
        for r, fds in got.items():
            for f_ in fds:
                os.close(f_)
        self.tensor(torch.uint8).zero_()
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier(self.group)

    def close(self) -> None:
        """Collective release (every rank of the group calls it, after the last kernel that touches the buffer has finished):
        unmap the multicast mapping and every peer mapping, drop the allocation handles.  Buffers normally live as long as the
        process; this exists for long-running services that rebuild plans (rpc/service.py plan cache eviction)."""
        if getattr(self, "_closed", False):
            return
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier(self.group)          # nobody unmaps pages a peer kernel may still be reading
        lib = self.lib
        if self.backend == "vmm":
            if self.mc_ptr is not None:
                lib.tepd_vmm_unmap(self.mc_ptr, self.nbytes)
                lib.tepd_vmm_release(self._mc_handle)
                self.mc_ptr = None
            for q, h in zip(self.ptrs, self._handles):
                lib.tepd_vmm_unmap(q, self.nbytes)
                lib.tepd_vmm_release(h)
        else:
            for r, q in enumerate(self.ptrs):
                if r != self.rank:
                    lib.tepd_ipc_close(q)
            if self.world > 1:
                dist.barrier(self.group)      # peers have closed their mappings before the owner frees
            lib.tepd_symm_free(self.local_ptr)
        self.ptrs, self._closed = [], True

    def tensor(self, dtype: torch.dtype, numel: Optional[int] = None, offset_bytes: int = 0) -> torch.Tensor:
        """Zero-copy torch view of the LOCAL buffer."""
        t = torch.as_tensor(_CudaArray(self.local_ptr + offset_bytes, self.nbytes - offset_bytes), device="cuda")
        t = t.view(dtype)
        return t if numel is None else t[:numel]


class McContext:
    """Flag state for the multimem kernels of ONE stream of launches: a symmetric flag word per CTA slot (signalled with a
    single `multimem.red` per rank), a local arrival count per slot (nothing is ever reset, so captured launches replay
    unchanged) and an error word that a timed-out spin raises instead of hanging the box."""

    MAX_CTAS = 512

    def __init__(self, group=None):
        self.flags = SymmetricBuffer(self.MAX_CTAS * 4, group, backend="vmm")
        if self.flags.mc_ptr is None:
            raise RuntimeError("multicast is not available in this group")
        self.lib = self.flags.lib
        self.world, self.rank = self.flags.world, self.flags.rank
        dev = torch.device("cuda", torch.cuda.current_device())
        self.epochs = torch.zeros(self.MAX_CTAS, dtype=torch.int32, device=dev)
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)

    def check(self) -> None:
        if int(self.err.item()):
            raise RuntimeError("a multimem barrier timed out: some rank never arrived")

    def barrier(self, stream: Optional[int] = None) -> None:
        s = torch.cuda.current_stream().cuda_stream if stream is None else stream
        rc = self.lib.tepd_mc_barrier(self.flags.mc_ptr, self.flags.local_ptr, self.epochs.data_ptr(), self.world,
                                      self.err.data_ptr(), s)
        if rc:
            raise RuntimeError(f"mc_barrier failed ({rc})")
        ops._count()

    def all_reduce_bf16_(self, buf: SymmetricBuffer, numel: int, N: int, bias: Optional[torch.Tensor] = None,
                         residual: Optional[torch.Tensor] = None, offset_bytes: int = 0, ctas: int = 0) -> None:
        """In place on the symmetric bf16 buffer: buf[:numel] <- sum over ranks (+ bias[col] + residual), on every rank.  One
        kernel: barrier, `multimem.ld_reduce` of this rank's 1/n slice, epilogue, `multimem.st` to all, barrier."""
        assert buf.mc_ptr is not None and numel % (8 * self.world) == 0
        rc = self.lib.tepd_mc_all_reduce_bf16(buf.mc_ptr + offset_bytes, self.flags.mc_ptr, self.flags.local_ptr,
                                              self.epochs.data_ptr(), self.world, self.rank, numel, N,
                                              None if bias is None else bias.data_ptr(),
                                              None if residual is None else residual.data_ptr(), self.err.data_ptr(), ctas,
                                              torch.cuda.current_stream().cuda_stream)
        if rc:
            raise RuntimeError(f"mc_all_reduce_bf16 failed ({rc})")
        ops._count()


class SymmBarrier:
    """Cross-rank barrier through peer memory (one tiny kernel; CUDA-graph capturable)."""

    def __init__(self, group=None):
        self.buf = SymmetricBuffer(256, group)
        self.epoch = torch.zeros(1, dtype=torch.int32, device="cuda")

    def __call__(self, stream: Optional[int] = None) -> None:
        s = torch.cuda.current_stream().cuda_stream if stream is None else stream
        rc = self.buf.lib.tepd_symm_barrier(self.buf.ptr_array, self.buf.world, self.buf.rank, self.epoch.data_ptr(), s)
        if rc:
            raise RuntimeError(f"symm_barrier failed ({rc})")
        ops._count()


class FusedShardedOptimizer:
    """reduce-scatter(grad) + AdamW(owned shard) + bf16 all-gather(param) as one kernel per bucket.

    Multicast-bound buffers (backend 'vmm'): the NVLS kernel -- the gradient chunk arrives already summed by the switch
    (`multimem.ld_reduce`, one load per 16 bytes instead of n-1 peer loads) and the updated bf16 shard leaves the GPU once
    (`multimem.st`, replicated by the switch instead of n-1 peer stores); barriers are one `multimem.red` per rank with a
    bounded spin.  Opt-in (TEPDIST_DP_MC=1): a reduce-scatter through the switch still costs every GPU its full gradient buffer
    in egress, so NVLS only pays for the all-gather half.  Default: unicast P2P loads / stores (IPC or VMM mappings alike)."""

    def __init__(self, grad_buf: SymmetricBuffer, param_buf: SymmetricBuffer, group=None, grad16_buf: Optional[SymmetricBuffer] = None):
        import os
        self.g, self.p = grad_buf, param_buf
        self.g16 = grad16_buf          # bf16 staging copy of the gradients (bf16 wire; implies the NVLS kernel)
        self.world, self.rank = grad_buf.world, grad_buf.rank
        self.mc: Optional[McContext] = None
        if (grad_buf.mc_ptr is not None and param_buf.mc_ptr is not None
                and (os.environ.get("TEPDIST_DP_MC", "0") == "1" or grad16_buf is not None)):
            self.mc = McContext(group)
            self._barrier = None
        else:
            self._barrier = SymmBarrier(group)
        self.mc_ctas = int(os.environ.get("TEPDIST_MC_CTAS", "0"))
        self.dry = False     # timing-only: same kernel on local memory alone (exposed-communication measurement)

    def barrier(self) -> None:
        if self.dry:
            return
        if self.mc is not None:
            self.mc.barrier()
        else:
            self._barrier()

    def step(self, master, m, v, begin: int, end: int, n_decay: int, hyper, beta1, beta2, eps, wd, ctas: int = 0,
             local_grad: bool = False) -> None:
        """local_grad: the gradient of [begin, end) is already complete on every rank (replicated computation): only the
        update is sharded -- the owner reads its local gradient and still stores the new bf16 values to every peer."""
        if self.mc is not None and not self.dry and not local_grad and begin % 8 == 0 and end % 8 == 0:
            src = self.g16 if self.g16 is not None else self.g
            rc = self.g.lib.tepd_mc_rs_adamw_ag(src.mc_ptr, self.p.mc_ptr, master.data_ptr(), m.data_ptr(), v.data_ptr(),
                                                begin, end, n_decay, beta1, beta2, eps, wd, hyper.data_ptr(),
                                                int(self.g16 is not None), self.mc_ctas or ctas,
                                                torch.cuda.current_stream().cuda_stream)
            if rc:
                raise RuntimeError(f"mc_rs_adamw_ag failed ({rc})")
            ops._count()
            return
        gp, pp, n = self.g.ptr_array, self.p.ptr_array, self.world
        n_grad = n
        if local_grad:
            gp, n_grad = (ctypes.c_void_p * 1)(self.g.local_ptr), 1
        if self.dry:
            gp, pp, n, n_grad = (ctypes.c_void_p * 1)(self.g.local_ptr), (ctypes.c_void_p * 1)(self.p.local_ptr), 1, 1
        rc = self.g.lib.tepd_fused_rs_adamw_ag(gp, pp, master.data_ptr(), m.data_ptr(), v.data_ptr(),
                                               n, begin, end, n_decay, beta1, beta2, eps, wd, hyper.data_ptr(), ctas,
                                               torch.cuda.current_stream().cuda_stream, n_grad)
        if rc:
            raise RuntimeError(f"fused_rs_adamw_ag failed ({rc})")
        ops._count()


# ------------------------------------------------------------------------------------------------ tensor-parallel fused GEMM
class GemmAllReduceMC:
    """Row-parallel linear + ALL-reduce over NVLS: the wgmma GEMM writes its bf16 partial [M, N] straight into a
    symmetric buffer (no staging copy), then ONE multimem kernel reduces it inside the NVSwitch -- every rank pulls its 1/n
    slice with `multimem.ld_reduce` (fp32 accumulation in the switch), adds bias + residual and publishes the finished
    rows to all ranks with `multimem.st`; the two cross-rank barriers live inside that kernel (one `multimem.red` per CTA).
    Per element the owner receives 1x (not (n-1)x) and sends 1x (not (n-1)x): the NVLink bytes of a tensor-parallel
    all-reduce no longer grow with n.  One instance serves every call site of a given [M, N]; each call site owns its
    symmetric output buffer, allocated with `new_output()`."""

    def __init__(self, M: int, N: int, group=None, ctx: Optional["McContext"] = None, ctas: int = 0):
        self.M, self.N, self.group = M, N, group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        assert (M * N) % (8 * self.world) == 0
        self.ctx = ctx or McContext(group)
        self.ctas = ctas

    def new_output(self) -> SymmetricBuffer:
        return SymmetricBuffer(self.M * self.N * 2, self.group, backend="vmm")

    def __call__(self, x: torch.Tensor, w: torch.Tensor, out: SymmetricBuffer, bias: Optional[torch.Tensor] = None,
                 residual: Optional[torch.Tensor] = None, b_mn: bool = False, block_n: int = 0) -> torch.Tensor:
        y = out.tensor(torch.bfloat16, self.M * self.N).view(self.M, self.N)
        ops.gemm(x, w, b_mn=b_mn, out=y)
        if residual is not None:
            assert residual.is_contiguous() and residual.dtype == torch.bfloat16
        self.ctx.all_reduce_bf16_(out, self.M * self.N, self.N, bias=bias, residual=residual, ctas=self.ctas)
        return y
