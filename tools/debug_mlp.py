"""GPU-side diagnostics of the wgmma MLP layer kernel (prints, does not assert)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from pvn3d_b200 import mlp, _ext

dev = torch.device("cuda:0")
torch.backends.cuda.matmul.allow_tf32 = False


def ref_dense(a, w, b, relu, pool):
    y = a.double() @ w.double().t() + b.double()
    if relu:
        y = y.clamp_min(0)
    if pool:
        y = y.view(-1, pool, y.size(-1)).max(1).values
    return y.float()


def check(name, got, want):
    err = (got - want).abs()
    scale = want.abs().mean().item() + 1e-9
    print(f"{name:60s} max_abs {err.max().item():.3e}  mean_abs {err.mean().item():.3e}  scale {scale:.3e}  "
          f"rel {err.max().item() / scale:.2e}", flush=True)
    return err


g = torch.Generator(device="cpu").manual_seed(0)
for (rows, k, n, relu, pool) in [(128, 32, 16, False, 0), (256, 32, 32, False, 0), (300, 64, 64, True, 0),
                                 (1000, 96, 128, True, 0), (512, 128, 208 - 12, True, 0), (512, 256, 384, True, 0),
                                 (640, 544, 256, True, 0), (2048, 384, 512, True, 32), (1024, 64, 32, True, 16),
                                 (256, 32, 16, False, 8)]:
    a = torch.randn(rows, k, generator=g)
    w = torch.randn(n, k, generator=g) / np.sqrt(k)
    b = torch.randn(n, generator=g)
    layer = mlp.PackedLayer(w.to(dev), b.to(dev))
    lda = (k + 15) // 16 * 16
    ad = torch.zeros(rows, lda, device=dev)
    ad[:, :k] = a.to(dev)
    try:
        out = mlp.mlp_dense(ad, layer, relu=relu, pool=pool)
        torch.cuda.synchronize()
    except Exception as e:
        print("FAIL", rows, k, n, e)
        continue
    want = ref_dense(mlp.tf32_round(a), mlp.tf32_round(w), b, relu, pool).to(dev)
    err = check(f"dense rows={rows} k={k} n={n} relu={relu} pool={pool}", out[:, :n], want)
    if err.max().item() > 1e-2 and rows <= 300:
        # structure of the error: which rows / cols are wrong
        bad = (err > 1e-2)
        print("   bad rows:", bad.any(1).nonzero().flatten()[:20].tolist(), " bad cols:", bad.any(0).nonzero().flatten()[:20].tolist())
    if out.size(1) > n:
        print("   pad cols max:", out[:, n:].abs().max().item())

# identity probe: A = one-hot rows, W = identity  -> out[p, n] = (p % k == n)
rows, k, n = 128, 32, 32
ad = torch.zeros(rows, k, device=dev)
ad[torch.arange(rows), torch.arange(rows) % k] = 1.0
layer = mlp.PackedLayer(torch.eye(n, k, device=dev) * torch.arange(1, n + 1, device=dev)[:, None], torch.zeros(n, device=dev))
out = mlp.mlp_dense(ad, layer, relu=False)
torch.cuda.synchronize()
want = ad @ (torch.eye(n, k, device=dev) * torch.arange(1, n + 1, device=dev)[:, None]).t()
print("identity probe max err", (out - want).abs().max().item())
if (out - want).abs().max().item() > 1e-3:
    print(out[:8, :8])

# FP first layer
from oracle import pn2
rng = np.random.default_rng(1)
b_, n_u, m_k, c2, c1 = 2, 512, 128, 256, 96
unk = rng.uniform(0, 1, (b_, n_u, 3)).astype(np.float32)
kn = rng.uniform(0, 1, (b_, m_k, 3)).astype(np.float32)
d2, nn = pn2.three_nn(unk, kn)
kf = rng.normal(size=(b_, m_k, c2)).astype(np.float32)
sk = rng.normal(size=(b_, n_u, c1)).astype(np.float32)
nw = mlp.three_nn_weights(torch.from_numpy(d2).to(dev))
dr = 1.0 / (torch.sqrt(torch.from_numpy(d2)) + 1e-8)
wref = dr / dr.sum(2, keepdim=True)
print("nn weights max diff", (nw.cpu() - wref).abs().max().item())
interp = (torch.from_numpy(kf)[torch.arange(b_)[:, None, None], torch.from_numpy(nn).long()] * wref[..., None]).sum(2)
X = torch.cat([interp, torch.from_numpy(sk)], -1).reshape(-1, c2 + c1)
w = (rng.normal(size=(128, c2 + c1)) / 16).astype(np.float32)
bias = rng.normal(size=128).astype(np.float32)
want = ref_dense(mlp.tf32_round(X), mlp.tf32_round(torch.from_numpy(w)), torch.from_numpy(bias), True, 0).to(dev)
layer = mlp.PackedLayer(torch.from_numpy(w).to(dev), torch.from_numpy(bias).to(dev))
skd = torch.from_numpy(sk).to(dev)
out = mlp.mlp_fp_first(torch.from_numpy(kf).to(dev), torch.from_numpy(nn).to(dev), nw, skd.data_ptr(), c1, c1, layer)
torch.cuda.synchronize()
check("fp_first c2=256 c1=96", out[:, :128], want)

# whole model vs golden
from pvn3d_b200 import testing
z = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests/golden/pn2msg.npz"))
model = testing.seeded_pointnet2msg(0, 1)
eng = mlp.FusedPointnet2MSG(model, dev)
x = torch.from_numpy(z["cld_rgb_nrm"])[None].to(dev)
y = eng(x)[0]
torch.cuda.synchronize()
got = y[:, torch.from_numpy(z["cols"]).long().to(dev)].cpu().numpy()
e = np.abs(got - z["feats"])
print("FusedPointnet2MSG vs reference golden: max", e.max(), "mean", e.mean(), "feature abs mean", float(z["feat_abs_mean"]))
import time
xb = x.repeat(32, 1, 1).contiguous() if False else None
