"""Accuracy probe of the wgmma 3xTF32 engine vs the fp32 SIMT engine against an fp64 reference (run on an H100)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rl_x_b200.algorithms.ppo.b200.kernels import PpoKernels

CASES = [(0, 0, 128, 128, 32), (0, 0, 128, 256, 64), (0, 1, 4096, 512, 376), (0, 1, 130, 256, 256), (0, 0, 1000, 128, 64), (0, 1, 32, 512, 376),
         (1, 0, 256, 256, 256), (1, 2, 4100, 256, 256), (1, 2, 33, 256, 256),
         (2, 0, 128, 128, 64), (2, 0, 256, 256, 3000), (2, 0, 512, 380, 2752), (2, 0, 512, 380, 40), (2, 0, 256, 256, 5)]


def _k():
    return PpoKernels(376, 17, 256)


def _err(c, ref):
    c, ref = c.double().cpu(), ref.cpu()
    return float((c - ref).norm() / ref.norm()), float((c - ref).abs().max() / ref.abs().max())


DEV='cuda'
k=_k()
extra=[(0,0,4096,512,376),(0,0,4096,256,256),(2,0,512,380,344),(2,0,512,380,1376),(2,0,512,380,32768),(2,0,256,256,928),(0,0,256,256,8192)]
for (layout,epi,M,N,K) in CASES+extra:
    g=torch.Generator().manual_seed(M*7+N*3+K)
    if layout==0: A,B=torch.randn(M,K,generator=g),torch.randn(N,K,generator=g)*0.3; ref=A.double()@B.double().T
    elif layout==1: A,B=torch.randn(M,K,generator=g),torch.randn(K,N,generator=g)*0.3; ref=A.double()@B.double()
    else: A,B=torch.randn(K,M,generator=g),torch.randn(K,N,generator=g)*0.3; ref=A.double().T@B.double()
    bias=torch.randn(N,generator=g) if epi==1 else None
    aux=torch.tanh(torch.randn(M,N,generator=g)) if epi==2 else None
    if epi==1: ref=torch.tanh(ref+bias.double())
    if epi==2: ref=ref*(1-aux.double()**2)
    res=[]
    for engine in (0,1):
        C=torch.full((M,N),float('nan'),device=DEV)
        k.debug_gemm(engine,layout,epi,A.to(DEV),B.to(DEV),C,M,N,K,bias=bias.to(DEV) if bias is not None else None,aux=aux.to(DEV) if aux is not None else None)
        torch.cuda.synchronize()
        fin=bool(torch.isfinite(C).all())
        e=_err(C,ref)
        # signed mean relative error of |C| vs |ref| (bias detection)
        sb=float(((C.double().cpu().abs()-ref.abs()).sum()/ref.abs().sum()))
        res.append((fin,e,sb))
    print(f"layout={layout} epi={epi} M={M} N={N} K={K} | simt fro={res[0][1][0]:.2e} max={res[0][1][1]:.2e} bias={res[0][2]:+.1e} | tc finite={res[1][0]} fro={res[1][1][0]:.2e} max={res[1][1][1]:.2e} bias={res[1][2]:+.1e}")
