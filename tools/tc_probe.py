"""Sweep descriptor conventions of the wgmma probe on a real H100 and print which are correct."""
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pocketflow_b200 import lib as _lib  # noqa: E402

L = _lib.load()
L.pf_tc_probe.restype = ctypes.c_int32
L.pf_tc_probe.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int32] * 3 + [ctypes.c_uint32] * 6 + [ctypes.c_void_p]


def run(mode, N, K, lbo_a, sbo_a, lbo_b, sbo_b, ks_a, ks_b):
    torch.manual_seed(0)
    if mode == 0:
        A = torch.randn(128, K, device='cuda').bfloat16()
        B = torch.randn(N, K, device='cuda').bfloat16()
        ref = A.float() @ B.float().t()
    else:
        A = torch.randn(K, 128, device='cuda').bfloat16()
        B = torch.randn(K, N, device='cuda').bfloat16()
        ref = A.float().t() @ B.float()
    D = torch.zeros(128, N, device='cuda')
    st = L.pf_tc_probe(A.data_ptr(), B.data_ptr(), D.data_ptr(), N, K, mode, lbo_a, sbo_a, lbo_b, sbo_b, ks_a, ks_b,
                       None)
    torch.cuda.synchronize()
    err = (D - ref).abs().max().item() / ref.abs().max().item()
    return st, err


if __name__ == '__main__':
    for N, K in ((128, 64), (128, 256), (64, 128), (256, 128), (16, 64)):
        for lbo in (0, 16, 1024):
            st, err = run(0, N, K, lbo, 1024, lbo, 1024, 32, 32)
            print('K-major  N=%3d K=%3d lbo=%4d sbo=1024 kstep=32 -> status %d err %.3e %s' % (
                N, K, lbo, st, err, 'OK' if err < 1e-5 else 'WRONG'), flush=True)
    for N, K in ((128, 64), (128, 256), (64, 128), (256, 128)):
        mbA, mbB = 128 // 64, N // 64
        cands = [
            ('lbo=mblk,sbo=kblk', 1024, mbA * 1024, 1024, mbB * 1024, 2 * mbA * 1024, 2 * mbB * 1024),
            ('lbo=kblk,sbo=mblk', mbA * 1024, 1024, mbB * 1024, 1024, 2 * mbA * 1024, 2 * mbB * 1024),
        ]
        for name, la, sa, lb, sb, ka, kb in cands:
            st, err = run(1, N, K, la, sa, lb, sb, ka, kb)
            print('MN-major N=%3d K=%3d %s -> status %d err %.3e %s' % (N, K, name, st, err,
                                                                        'OK' if err < 1e-5 else 'WRONG'), flush=True)
