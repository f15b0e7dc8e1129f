"""Dynamic Sequence Parallelism communication -- host-side mirror of videosys/core/distributed/comm.py.

Same function names / argument meaning as the reference (set_pad/get_pad :268-279, split_sequence /
gather_sequence :148-190,256-261, all_to_all_with_pad :282-304, all_to_all_comm :139-140,
split/gather_from_second_dim :307-318), inference only (no autograd functions); ``ulysses_scatter_heads`` /
``ulysses_gather_heads`` are CogVideoX's head-scatter exchange on the packed qkv (cogvideox_transformer_3d.py:44-165).

Two transports for the dimension switch:
  * ``DspP2P`` (native path): the switch is fused into its producer and consumer kernels.  The modulate kernel stores
    its rows straight into the owners' receive windows over NVLink (CUDA-IPC mapped peer memory), and the gate +
    residual kernel loads the branch back from the peers' windows; flags + a wait kernel order the streams; no staging
    copies, no NCCL launch (csrc/elementwise.cu, csrc/dsp_p2p.cu; C-ABI vsb_ln_modulate_dsp / vsb_gate_residual_dsp /
    vsb_dsp_signal / vsb_dsp_wait).
  * ``torch.distributed.all_to_all_single`` (NCCL on GPU, gloo on CPU for the host-logic tests): the fallback
    north_star allows "where the fused P2P kernel is not taken", and the only transport where CUDA IPC is unavailable.
"""
import ctypes as C
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

PAD_DICT: Dict[str, int] = {}


def set_pad(name: str, dim_size: int, parallel_group) -> None:
    sp = dist.get_world_size(parallel_group)
    PAD_DICT[name] = (sp - (dim_size % sp)) % sp


def get_pad(name: str) -> int:
    return PAD_DICT[name]


def _append(x: torch.Tensor, dim: int, n: int, value: float = 0.0) -> torch.Tensor:
    shape = list(x.shape)
    shape[dim] = n
    return torch.cat([x, x.new_full(shape, value)], dim=dim)


def split_sequence(input_, process_group, dim, grad_scale=1.0, pad=0, pad_val=0):
    """This rank's equal chunk along ``dim`` after appending ``pad`` entries of ``pad_val`` (no communication)."""
    world = dist.get_world_size(process_group)
    if world == 1:
        return input_
    if pad > 0:
        input_ = _append(input_, dim, pad, pad_val)
    size = input_.size(dim)
    assert size % world == 0, f"dim_size ({size}) is not divisible by world_size ({world})"
    step = size // world
    rank = dist.get_rank(process_group)
    return input_.narrow(dim, rank * step, step).contiguous()


def gather_sequence(input_, process_group, dim, grad_scale=1.0, pad=0):
    """all_gather along ``dim`` then drop the trailing ``pad`` entries."""
    world = dist.get_world_size(process_group)
    input_ = input_.contiguous()
    if world == 1:
        return input_
    parts = [torch.empty_like(input_) for _ in range(world)]
    dist.all_gather(parts, input_, group=process_group)
    out = torch.cat(parts, dim=dim)
    return out.narrow(dim, 0, out.size(dim) - pad) if pad > 0 else out


def all_to_all_comm(input_, process_group=None, scatter_dim=2, gather_dim=1):
    """Scatter ``scatter_dim`` / gather ``gather_dim`` across the group with one all_to_all_single."""
    world = dist.get_world_size(process_group)
    if world == 1:
        return input_
    assert input_.shape[scatter_dim] % world == 0
    # [.., world, chunk, ..] -> leading 'destination rank' axis, contiguous send buffer
    send = torch.stack(torch.tensor_split(input_, world, scatter_dim), dim=0).contiguous()
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=process_group)
    return torch.cat(list(recv.unbind(0)), dim=gather_dim).contiguous()


def all_to_all_with_pad(input_, process_group, scatter_dim: int = 2, gather_dim: int = 1, scatter_pad: int = 0,
                        gather_pad: int = 0):
    if scatter_pad > 0:
        input_ = _append(input_, scatter_dim, scatter_pad, 0.0)
    world = dist.get_world_size(process_group)
    assert input_.shape[scatter_dim] % world == 0, (
        f"Dimension to scatter ({input_.shape[scatter_dim]}) is not divisible by world size ({world})"
    )
    out = all_to_all_comm(input_, process_group, scatter_dim, gather_dim)
    if gather_pad > 0:
        out = out.narrow(gather_dim, 0, out.size(gather_dim) - gather_pad)
    return out


def split_from_second_dim(x, batch_size, parallel_group):
    x = x.view(batch_size, -1, *x.shape[1:])
    x = split_sequence(x, parallel_group, dim=1, grad_scale="down", pad=get_pad("temporal"))
    return x.reshape(-1, *x.shape[2:])


def gather_from_second_dim(x, batch_size, parallel_group):
    x = x.view(batch_size, -1, *x.shape[1:])
    x = gather_sequence(x, parallel_group, dim=1, grad_scale="up", pad=get_pad("temporal"))
    return x.reshape(-1, *x.shape[2:])


def ulysses_scatter_heads(qkv: torch.Tensor, n_text: int, process_group) -> torch.Tensor:
    """Head-scatter all-to-all of CogVideoX's joint attention (reference cogvideox_transformer_3d.py:112-122 followed by
    ``_remove_extra_encoder`` :44-62), on the PACKED projection.

    qkv: [B, n_text + Nl, 3, H, D] -- this rank's rows (the replicated text rows, then its 1/world chunk of the video
    rows), every head.  Returns [B, n_text + world * Nl, 3, H / world, D]: every row, this rank's head group.  The
    reference ships the text rows to every peer and drops all copies but the first; each rank already holds those rows
    (computed from the replicated text stream), so only the video rows travel: one ``all_to_all_single``."""
    world = dist.get_world_size(process_group)
    rank = dist.get_rank(process_group)
    B, L, three, H, D = qkv.shape
    assert H % world == 0, f"Number of heads {H} must be divisible by sequence parallel size {world}"
    Hn, Nl = H // world, L - n_text
    send = qkv[:, n_text:].reshape(B, Nl, three, world, Hn, D).permute(3, 0, 1, 2, 4, 5).contiguous()
    recv = torch.empty_like(send)  # [source rank, B, Nl, 3, Hn, D]
    dist.all_to_all_single(recv, send, group=process_group)
    out = qkv.new_empty(B, n_text + world * Nl, three, Hn, D)
    out[:, :n_text] = qkv[:, :n_text, :, rank * Hn : (rank + 1) * Hn]
    out[:, n_text:].view(B, world, Nl, three, Hn, D).copy_(recv.permute(1, 0, 2, 3, 4, 5))
    return out


def ulysses_gather_heads(o: torch.Tensor, n_text: int, process_group) -> torch.Tensor:
    """The way back (reference :162-165: ``_add_extra_encoder`` then all_to_all scatter rows / gather heads).

    o: [B, n_text + world * Nl, Hn * D] -- every row, this rank's heads.  Returns [B, n_text + Nl, world * Hn * D]: the
    text rows and this rank's video rows with every head (head group g in columns [g * Hn * D, (g + 1) * Hn * D))."""
    world = dist.get_world_size(process_group)
    B, L, Cn = o.shape
    Nl = (L - n_text) // world
    send = torch.empty(world, B, n_text + Nl, Cn, dtype=o.dtype, device=o.device)
    send[:, :, :n_text] = o[:, :n_text]  # the text rows go to every peer (the reference's "extra encoder")
    send[:, :, n_text:] = o[:, n_text:].view(B, world, Nl, Cn).transpose(0, 1)
    recv = torch.empty_like(send)  # [head group, B, n_text + Nl, Cn]
    dist.all_to_all_single(recv, send, group=process_group)
    return recv.permute(1, 2, 0, 3).reshape(B, n_text + Nl, world * Cn)


class DspP2P:
    """Symmetric receive windows + flags for the P2P dimension switch (one instance per process / sp group).

    The native replacement of STDiT3Block.dynamic_switch (open_sora_transformer_3d.py:288-315):
    ``ln_modulate_push`` is the S-shard -> T-shard switch fused into the modulate kernel, ``branch_window`` +
    ``gate_residual_pull`` the way back fused into the gate + residual kernel.  The two directions own separate windows
    and flag arrays; stream order plus the data dependencies of the block make one window per direction sufficient
    (see DESIGN.md section 5).
    """

    def __init__(self, process_group, max_elems: int, device: torch.device):
        from ... import _lib

        self._libmod = _lib
        self.lib = _lib.load()
        self.group = process_group
        self.world = dist.get_world_size(process_group)
        self.rank = dist.get_rank(process_group)
        self.device = device
        self.max_elems = int(max_elems)
        # epochs live on the DEVICE (flag slots 32 / 33, csrc/dsp_common.cuh): every call passes epoch = 0, so a
        # captured CUDA graph of a denoising step advances them on replay without the host
        self._own = []
        self._peer_recv: List[List[int]] = [[], []]
        self._peer_flag: List[List[int]] = [[], []]
        self._opened = []
        handles = []
        for d in range(2):
            buf = C.c_void_p()
            _lib.check(self.lib.vsb_dsp_alloc(C.byref(buf), self.max_elems * 2), "dsp_alloc")
            flg = C.c_void_p()
            _lib.check(self.lib.vsb_dsp_alloc(C.byref(flg), 64 * 4), "dsp_alloc")
            self._own.append((buf.value, flg.value))
            hb, hf = C.create_string_buffer(64), C.create_string_buffer(64)
            _lib.check(self.lib.vsb_ipc_get_handle(buf, hb), "ipc_get_handle")
            _lib.check(self.lib.vsb_ipc_get_handle(flg, hf), "ipc_get_handle")
            handles.append((hb.raw, hf.raw))
        everyone: List[Optional[list]] = [None] * self.world
        dist.all_gather_object(everyone, handles, group=process_group)
        for d in range(2):
            for r in range(self.world):
                if r == self.rank:
                    self._peer_recv[d].append(self._own[d][0])
                    self._peer_flag[d].append(self._own[d][1])
                    continue
                pb, pf = C.c_void_p(), C.c_void_p()
                _lib.check(self.lib.vsb_ipc_open_handle(everyone[r][d][0], C.byref(pb)), "ipc_open_handle")
                _lib.check(self.lib.vsb_ipc_open_handle(everyone[r][d][1], C.byref(pf)), "ipc_open_handle")
                self._opened += [pb.value, pf.value]
                self._peer_recv[d].append(pb.value)
                self._peer_flag[d].append(pf.value)
        self._recv_arr = [(C.c_void_p * self.world)(*self._peer_recv[d]) for d in range(2)]
        self._flag_arr = [(C.c_void_p * self.world)(*self._peer_flag[d]) for d in range(2)]
        dist.barrier(group=process_group)

    def _window(self, d: int, shape) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= s
        assert n <= self.max_elems, "DSP window too small"
        from ..._cuda_view import device_view

        return device_view(self._own[d][0], shape, torch.bfloat16, self.device)

    # ---- producer- / consumer-fused switch (csrc/elementwise.cu: ln_modulate_kernel<.., true>, gate_residual_dsp_kernel)
    def ln_modulate_push(self, x, mod, mask_u8, shift_row: int, scale_row: int, B: int, T: int, Sl: int, Sg: int,
                         eps: float = 1e-6) -> torch.Tensor:
        """AdaLN modulate of the local S-shard x [B, T*Sl, C] whose stores ARE the S-shard -> T-shard switch: returns
        this rank's receive window as [1, Tl, Sg, C] (the (batch, frame) sequences it owns, every patch of each)."""
        from ... import kernels

        w, Cc = self.world, x.shape[-1]
        Tl = -(-(B * T) // w)
        st = torch.cuda.current_stream().cuda_stream
        with kernels._Timed("dsp_push", x.numel() * 2 * (w - 1) // w):
            self._libmod.check(
                self.lib.vsb_ln_modulate_dsp(x.data_ptr(), mod.data_ptr(), None if mask_u8 is None else mask_u8.data_ptr(),
                                             shift_row, scale_row, B, T, Sl, Cc, eps, self._recv_arr[0], self._flag_arr[0],
                                             self.rank, w, Sg, 0, st),
                "ln_modulate_dsp",
            )
            self._libmod.check(self.lib.vsb_dsp_wait(self._own[0][1], w, 0, st), "dsp_wait")
        return self._window(0, (1, Tl, Sg, Cc))

    def branch_window(self, B: int, T: int, Sg: int, Cc: int) -> torch.Tensor:
        """This rank's OWN direction-1 window as [Tl * Sg, C]: the proj GEMM writes the attention branch here and the
        peers pull their columns from it (gate_residual_pull)."""
        Tl = -(-(B * T) // self.world)
        return self._window(1, (Tl * Sg, Cc))

    def gate_residual_pull(self, x, mod, mask_u8, gate_row: int, B: int, T: int, Sl: int, Sg: int, out=None,
                           cache_out=None) -> torch.Tensor:
        """Publishes 'my branch window is written', waits for every peer's, then x + gate * y with y PULLED over
        NVLink from the owners' windows (the T-shard -> S-shard switch fused into the consumer's loads)."""
        from ... import kernels

        w, Cc = self.world, x.shape[-1]
        st = torch.cuda.current_stream().cuda_stream
        out = torch.empty_like(x) if out is None else out
        with kernels._Timed("dsp_pull", x.numel() * 2 * (w - 1) // w):
            self._libmod.check(self.lib.vsb_dsp_signal(self._flag_arr[1], self.rank, w, 0, st), "dsp_signal")
            self._libmod.check(self.lib.vsb_dsp_wait(self._own[1][1], w, 0, st), "dsp_wait")
            self._libmod.check(
                self.lib.vsb_gate_residual_dsp(x.data_ptr(), self._recv_arr[1], out.data_ptr(),
                                               None if cache_out is None else cache_out.data_ptr(), mod.data_ptr(),
                                               None if mask_u8 is None else mask_u8.data_ptr(), gate_row, B, T, Sl, Cc,
                                               self.rank, w, Sg, st),
                "gate_residual_dsp",
            )
        return out

    def close(self):
        for p in self._opened:
            self.lib.vsb_ipc_close_handle(p)
        self._opened = []
        for buf, flg in self._own:
            self.lib.vsb_dsp_free(buf)
            self.lib.vsb_dsp_free(flg)
        self._own = []
