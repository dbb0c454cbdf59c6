"""GPU debug aid: run the tensor-core linear op on structured inputs and dump outputs + references so descriptor /
swizzle mistakes can be diagnosed offline from one gpurun call.  Writes gpurun_out/linear_debug.npz."""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))
from mvb200 import _lib  # noqa: E402

lib = _lib.load()
out = {}
st = C.c_void_p(0)
cases = [("t128_k64", 128, 64, 2, 0, 1), ("t128_k64_lo", 128, 64, 2, 1, 1), ("t128_k256", 128, 256, 3, 1, 1),
         ("t256_k256_s2", 256, 256, 3, 1, 2), ("t384_k2048_auto", 384, 2048, 16, 1, 0), ("v2562_k2048", 2562, 2048, 5, 1, 0)]
for name, M, K, R, lo, ks in cases:
    g = torch.Generator().manual_seed(1)
    W = (torch.randn(M, K, generator=g) * 0.1).to(torch.bfloat16)
    x = torch.randn(R, K, generator=g)
    if name == "t128_k64":
        # identity-like probe: W[j, k] = 1 if k == j % 64 ; x[n, k] = k + 100 n  -> y[n, j] = (j % 64) + 100 n
        W = torch.zeros(M, K); W[torch.arange(M), torch.arange(M) % K] = 1.0; W = W.to(torch.bfloat16)
        x = (torch.arange(K).float()[None, :] + 100.0 * torch.arange(R).float()[:, None])
    Wd, xd = W.cuda(), x.cuda()
    y = torch.full((R, M), -777.0, device="cuda")
    try:
        rc = lib.mvb_linear(Wd.data_ptr(), M, K, xd.data_ptr(), K, R, None, 1e-5, lo, ks, y.data_ptr(), M, 0, st)
        torch.cuda.synchronize()
        msg = lib.mvb_last_error().decode() if rc else "ok"
    except Exception as e:  # noqa: BLE001
        msg = f"exception {e}"
        rc = -1
    ref = (x.double() @ W.double().t()).float()
    got = y.cpu() if rc == 0 else torch.full((R, M), float("nan"))
    err = float((got - ref).abs().max() / ref.abs().max()) if rc == 0 else float("nan")
    print(f"{name}: rc={rc} {msg} rel_err={err:.3e}", flush=True)
    out[name + "_got"] = got.numpy(); out[name + "_ref"] = ref.numpy()
    if rc != 0:
        break
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
np.savez_compressed(os.path.join(ROOT, "gpurun_out", "linear_debug.npz"), **out)
