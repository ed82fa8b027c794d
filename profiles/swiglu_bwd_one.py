import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opendiloco_b200.ops import tc_gemm as T
M, I, Kd = 32768, 2688, 1024
dy = torch.randn(M, Kd, device="cuda").to(torch.bfloat16)
w_down = (torch.randn(Kd, I, device="cuda") * 0.05).to(torch.bfloat16)     # forward layout [h, I]
gu = torch.randn(M, 2 * I, device="cuda").to(torch.bfloat16)
for _ in range(3): T.linear_swiglu_bwd(dy, w_down, gu)
torch.cuda.synchronize()
