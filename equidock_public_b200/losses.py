"""Device-side training losses (csrc/losses.cu) behind a small host API: the reference's per-pair MSE, exact-EMD pocket OT
loss and body-intersection loss (src/train.py:41-49, 112-150; src/utils/ot_utils.py:5-29) with their gradients w.r.t. the
model outputs -- no per-pair D2H/H2D round trip through a CPU solver."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Sequence

import torch

from . import _native as nat


class PocketBatch:
    """Ragged per-pair targets of a batch on the device: bound ligand / receptor C-alpha coordinates (concatenated in batch
    order) and the pocket point pairs (``pocket_coors_ligand_list`` / ``pocket_coors_receptor_list``, src/train.py:118-119)."""

    def __init__(self, bound_lig: Sequence[torch.Tensor], bound_rec: Sequence[torch.Tensor],
                 pocket_lig: Sequence[torch.Tensor], pocket_rec: Sequence[torch.Tensor], device):
        f = lambda ts: torch.cat([t.reshape(-1, 3) for t in ts]).to(device=device, dtype=torch.float32).contiguous()
        self.bound_lig, self.bound_rec = f(bound_lig), f(bound_rec)
        self.pocket_lig, self.pocket_rec = f(pocket_lig), f(pocket_rec)
        sizes = [int(t.shape[0]) for t in pocket_lig]
        assert sizes == [int(t.shape[0]) for t in pocket_rec]
        ptr = [0]
        for s in sizes:
            ptr.append(ptr[-1] + s)
        self.n_pocket_total = ptr[-1]
        self.max_pocket = max(sizes) if sizes else 0
        self.pocket_ptr = torch.tensor(ptr, dtype=torch.int32, device=device)

    @classmethod
    def from_device_arrays(cls, bound_lig: torch.Tensor, bound_rec: torch.Tensor, pocket_lig: torch.Tensor,
                           pocket_rec: torch.Tensor, pocket_ptr: torch.Tensor, pocket_sizes: Sequence[int]) -> 'PocketBatch':
        """Over arrays already on the device in this class's layout (f32 (n,3) contiguous, ``pocket_ptr`` (B+1,) int32):
        no copy, no sync.  ``pocket_sizes`` are the per-pair pocket sizes, known on the host."""
        self = cls.__new__(cls)
        self.bound_lig, self.bound_rec, self.pocket_lig, self.pocket_rec = bound_lig, bound_rec, pocket_lig, pocket_rec
        sizes = [int(s) for s in pocket_sizes]
        self.n_pocket_total = sum(sizes)
        self.max_pocket = max(sizes) if sizes else 0
        self.pocket_ptr = pocket_ptr
        return self


def device_losses(plan, pred_lig: torch.Tensor, keypts: torch.Tensor, tgt: PocketBatch, pocket_ot_loss_weight: float,
                  intersection_loss_weight: float, intersection_sigma: float, intersection_surface_ct: float) -> Dict:
    """-> {'total': (4,) f64 [loss, mse, ot, intersection], 'parts': (B,4) f64, 'dcoors': (N_l,3) f32,
    'dkeypts': (2B,50,3) f64, 'plan': (n_pocket_total,50) i32, 'err': (1,) i32}.  'plan' is a view of the workspace
    holding the integer transport plans (pair b: rows pocket_ptr[b]..pocket_ptr[b+1], units of 1/(N_pocket * 50); rows of
    a pair the solver skipped are undefined).  check_loss_status(res) raises if a pocket exceeds the solver's capacity or
    the transport solve failed."""
    lib = nat.load()
    dev = pred_lig.device
    B, N_l = plan.n_pairs, plan.N_l
    assert pred_lig.shape == (N_l, 3) and tgt.bound_lig.shape == (N_l, 3) and tgt.bound_rec.shape == (plan.N_r, 3)
    with torch.cuda.device(dev):
        st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        ws_bytes = int(lib.eqd_losses_workspace_bytes(plan.N_r, tgt.n_pocket_total))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        parts = torch.zeros(B, 4, dtype=torch.float64, device=dev)
        total = torch.zeros(4, dtype=torch.float64, device=dev)
        dco = torch.empty(N_l, 3, dtype=torch.float32, device=dev)
        dkp = torch.empty(2 * B, nat.HEADS, 3, dtype=torch.float64, device=dev)
        err = torch.zeros(1, dtype=torch.int32, device=dev)
        pred = pred_lig.detach().to(torch.float32).contiguous()
        kp = keypts.detach().to(torch.float64).contiguous()
        nat.check(lib.eqd_losses(C.byref(plan.struct), nat.ptr(pred), nat.ptr(tgt.bound_lig), nat.ptr(tgt.bound_rec), nat.ptr(kp),
                                 nat.ptr(tgt.pocket_ptr), nat.ptr(tgt.pocket_lig), nat.ptr(tgt.pocket_rec), tgt.n_pocket_total,
                                 tgt.max_pocket, float(pocket_ot_loss_weight), float(intersection_loss_weight), float(intersection_sigma),
                                 float(intersection_surface_ct), nat.ptr(ws), ws_bytes, nat.ptr(parts), nat.ptr(total),
                                 nat.ptr(dco), nat.ptr(dkp), nat.ptr(err), st), 'eqd_losses')
    off = (max(plan.N_r, 1) * 8 + 255) // 256 * 256                     # plan_flow offset (eqd_iegmn.h)
    flow = ws[off:off + tgt.n_pocket_total * nat.HEADS * 4].view(torch.int32).view(tgt.n_pocket_total, nat.HEADS)
    return {'total': total, 'parts': parts, 'dcoors': dco, 'dkeypts': dkp, 'plan': flow, 'err': err,
            '_keep': (ws, pred, kp)}


def check_loss_status(res):
    e = int(res['err'].item())
    if e:
        raise nat.NativeLibraryError(f'eqd_losses: solver status {e} (1: pocket > 1024 points; other bits: transport solve failed)')
