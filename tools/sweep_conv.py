"""Time the modulated-conv kernel alone (hf_conv_time_kernel: CUDA events around N back-to-back launches, styles
and tables precomputed) over a ladder of generator layer shapes and batch sizes.  Prints algorithmic TFLOP/s
and the tiling plan.  Usage: python tools/sweep_conv.py [B ...]"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from hairfastgan_b200 import _lib
import hairfastgan_b200.model as M

torch.set_grad_enabled(False)
dev = torch.device("cuda", 0)
lib = _lib.lib()
LAYERS = [(512, 512, 16, 0), (512, 512, 16, 1), (512, 512, 32, 0), (512, 512, 32, 1), (512, 512, 64, 0),
          (512, 256, 64, 1), (256, 256, 128, 0), (256, 128, 128, 1), (128, 128, 256, 0), (128, 64, 256, 1),
          (64, 64, 512, 0), (64, 32, 512, 1), (32, 32, 1024, 0)]
batches = [int(a) for a in sys.argv[1:]] or [4, 12]
for (cin, cout, r, up) in LAYERS:
    m = M.StyledConv(cin, cout, 3, 512, upsample=bool(up)).to(dev)
    conv = m.conv
    desc, blob = conv._packed.get(conv, M.default_dtype())
    for B in batches:
        ro = 2 * r if up else r
        if B * cout * ro * ro * 4 > 6e9:
            continue
        x = torch.randn(B, cin, r, r, device=dev); st = torch.randn(B, 512, device=dev)
        y = torch.empty(B, cout, ro, ro, device=dev)
        ws = torch.empty(lib.hf_conv_workspace_bytes(C.byref(desc), B, r, r), dtype=torch.uint8, device=dev)
        io = _lib.hf_conv_io()
        io.batch, io.height, io.width = B, r, r
        io.x, io.style, io.style_dim, io.style_stride = x.data_ptr(), st.data_ptr(), 512, 512
        io.mod_weight, io.mod_bias, io.demodulate = conv.modulation.weight.data_ptr(), conv.modulation.bias.data_ptr(), 1
        io.y, io.workspace = y.data_ptr(), ws.data_ptr()
        ms = C.c_float(0)
        _lib.check(lib.hf_conv_time_kernel(C.byref(desc), blob.data_ptr(), C.byref(io), 10, C.byref(ms),
                                           torch.cuda.current_stream().cuda_stream), "time")
        plan = (C.c_int * 12)()
        lib.hf_conv_plan_query(C.byref(desc), B, r, r, plan)
        gf = 2.0 * cin * cout * 9 * r * r * B / 1e9
        print(f"{cin:4d}->{cout:4d} r={r:4d} up={up} B={B:3d}  {ms.value * 1e3:8.1f} us  {gf / ms.value:8.1f} TFLOP/s alg"
              f"  plan(0,n_tile,n_n,1,a_slots,0,0,stages,smem,work,grid,kc)={list(plan)}", flush=True)
        del x, y, ws
