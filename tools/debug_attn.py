"""dump the raw logits of the first key tile of the tensor-core attention kernel (debugging aid)

CTA (0,0,0) writes logits 0..15 (keys 0..15, before bias and scale) of query rows r with r % 16 < 8 into a [128, 40] buffer; they
are printed next to q . k of the same rows.  usage: python tools/debug_attn.py [head dim: 32 | 48 | 64]"""
import ctypes as C, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_util import OpRunner, ptr, view
from mug_diffusion_b200.engine import OpList
torch.manual_seed(0)
B, H, D, Lq, Lk = 1, 8, int(sys.argv[1]) if len(sys.argv) > 1 else 32, 48, 48
Cc = H * D
q, k, v = torch.randn(B, Lq, Cc), torch.randn(B, Lk, Cc), torch.randn(B, Lk, Cc)
rel, cg = torch.zeros(129, H), torch.ones(129, H)
R = OpRunner()
qc, kc, vc = q.reshape(-1, Cc).cuda(), k.reshape(-1, Cc).cuda(), v.reshape(-1, Cc).cuda()
out = torch.zeros(B * Lq, Cc).cuda()
dbg = torch.zeros(128 * 40).cuda()
R.lib.mugd_debug_set_attention_dump.argtypes = [C.c_void_p]
R.lib.mugd_debug_set_attention_dump(dbg.data_ptr())
ops = OpList()
relc, cgc = rel.cuda(), cg.cuda()
ops.attention(view(qc), view(kc), view(vc), view(out), ptr(relc), ptr(cgc), B, H, Lq, Lk, 64)
try:
    R.run(ops)
finally:
    R.lib.mugd_debug_set_attention_dump(None)
d = dbg.cpu().view(128, 40)
S_ref = q[0, :, :D].double() @ k[0, :, :D].double().t()
for r in (0, 5, 16, 37):
    print(f"row {r:2d} kernel:", [round(x, 5) for x in d[r, :16].tolist()])
    print(f"row {r:2d} ref   :", [round(x, 5) for x in S_ref[r, :16].tolist()])
print("max |kernel - ref| over the dumped logits:", float((d[[r for r in range(Lq) if r % 16 < 8], :16].double()
                                                         - S_ref[[r for r in range(Lq) if r % 16 < 8], :16]).abs().max()))
