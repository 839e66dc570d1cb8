"""Diagnostic sweep of the tensor-core conv kernels vs the oracle (prints errors, never asserts)."""
import os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import oracle as o
import caffe_mpi_b200 as m
from caffe_mpi_b200 import capi
from cases import ALL_CASES, make, tensors, rel_err

only = sys.argv[1:] 
rng = np.random.default_rng(1701)
dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
bad = 0
for name, case in ALL_CASES:
    if only and not any(s in name for s in only):
        continue
    po, pc = make(o, case), make(capi, case)
    x, w, b, dy = tensors(rng, po)
    wy = o.conv_forward(po, x, w, b, acc64=True)
    wdw, wdb, wdx = o.conv_backward(po, x, w, dy, acc64=True)
    for math in (capi.MATH_FP32, capi.MATH_TF32):
        d = m.ConvDesc(pc, capi.ENGINE_DEFAULT, math=math, algo=capi.ALGO_AUTO)
        algos = [d.algo_used(op) for op in (0, 1, 2)]
        X, W, B, DY = dev(x), dev(w), dev(b), dev(dy)
        Y = torch.full(po.y_shape(), 3.0, device="cuda"); DX = torch.full(po.x_shape(), 3.0, device="cuda")
        DW = torch.zeros(po.w_shape(), device="cuda")
        try:
            d.forward(X, W, B, Y); d.backward_data(DY, W, DX); d.backward_filter(X, DY, DW)
            torch.cuda.synchronize()
            e = [rel_err(Y.cpu().numpy(), wy), rel_err(DX.cpu().numpy(), wdx), rel_err(DW.cpu().numpy(), wdw)]
        except Exception as ex:
            e = [str(ex)]
        tol = 2e-5 if math == capi.MATH_FP32 else 1e-3
        flag = "" if all(isinstance(v, float) and v < tol for v in e) else "   <<<<<< FAIL"
        bad += bool(flag)
        print(f"{name:28s} math={math} algos={algos} err(y,dx,dw)={['%.2e' % v if isinstance(v, float) else v for v in e]}{flag}", flush=True)
print("FAILS:", bad)
