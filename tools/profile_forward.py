"""Run a few eager (un-graphed) forwards of a synthetic quantized ResNet so that ncu can capture individual launches.
   ncu --set full --import-source on --clock-control none -k regex:conv_igemm -s <skip> -c <n> -o prof python tools/profile_forward.py"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import hawq_b200 as hb  # noqa: E402
from hawq_b200 import qtensor  # noqa: E402
from hawq_b200.qtensor import IntActivation, Node  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--arch", default="resnet50")
ap.add_argument("--scheme", default="uniform8")
ap.add_argument("--batch", type=int, default=128)
ap.add_argument("--forwards", type=int, default=2)
ap.add_argument("--residual-bits", type=int, default=16)
a = ap.parse_args()
q = hb.build_synthetic_qresnet(a.arch, a.scheme, calib_batch=2)
s_in = float(q.quant_input.current_scale())
x = torch.clamp(torch.round(torch.randn(a.batch, 224, 224, 3) / s_in), -128, 127).to(torch.int8).cuda()
with torch.no_grad(), qtensor.engine_mode(residual_bits=a.residual_bits, checked=True):
    for _ in range(a.forwards):
        n, h, w, c = x.shape
        out = q(IntActivation(Node("int", (n, c, h, w), data=x.view(-1), bits=8, signed=True), x.device))
torch.cuda.synchronize()
print("done", out.shape)
