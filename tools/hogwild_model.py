#!/usr/bin/env python
"""CPU model of the fused kernel's parallelism at BASELINE config 2 (what the GPU parity numbers should look like).

Triples are visited in the order the kernel's 7104 lane groups retire them; the item rows of a WINDOW of 4 x 7104
triples (the rows a lane group has in flight) are read before any of the window's item deltas
land (stale reads), P[u] is sequential inside a lane group as in the kernel, item deltas are summed at the end of
the window.  float64, so what is measured is the schedule, not rounding.  Build-container result (about 4 min):
    loss rel 4.7e-06 | P max-norm rel 1.6e-03, rms err / rms update 1.8 % | Q max-norm rel 6.3e-03, 2.4 %
-- the same as re-ordering alone (tools/order_sensitivity.py): staleness inside the window is second order."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
rng=np.random.default_rng(0)
U,I,deg,d=1_000_000,100_000,50,64
lr,ru,ri=0.01,0.001,0.001
P0=(rng.random((U,d),dtype=np.float32)/3).astype(np.float64); Q0=(rng.random((I,d),dtype=np.float32)/3).astype(np.float64)
u=np.repeat(np.arange(U,dtype=np.int32),deg); i=rng.integers(0,I,U*deg,dtype=np.int32); j=((i+1+rng.integers(0,I-1,U*deg,dtype=np.int32))%I).astype(np.int32)
n=U*deg; G=7104; CH=32; INF=4
rounds=(n//CH)//G
main=np.arange(rounds*G*CH,dtype=np.int64).reshape(rounds,G,CH).transpose(0,2,1).reshape(-1)
perm=np.concatenate([main,np.arange(rounds*G*CH,n,dtype=np.int64)])
up,ip,jp=u[perm],i[perm],j[perm]
t0=time.time()
Pr,Qr,lref,_=bench.oracle_epoch(P0,Q0,u,i,j,np.float64)
print('oracle',time.time()-t0,flush=True)
P,Q=P0.copy(),Q0.copy(); loss=0.0
au,ai=lr*ru,lr*ri
W=G*INF
t0=time.time()
for w0 in range(0,n,W):
    sl=slice(w0,min(n,w0+W))
    uu,ii,jj=up[sl],ip[sl],jp[sl]
    qi=Q[ii]; qj=Q[jj]        # stale item rows for the whole window
    dQi=np.empty_like(qi); dQj=np.empty_like(qj)
    for t in range(0,len(uu),G):
        s2=slice(t,min(len(uu),t+G))
        p=P[uu[s2]]
        x=(p*qi[s2]).sum(1)-(p*qj[s2]).sum(1)
        s=1/(1+np.exp(-x)); g=(lr*(1-s))[:,None]
        pn=p+g*(qi[s2]-qj[s2])
        qin=qi[s2]+g*pn; qjn=qj[s2]-g*pn
        dp=(pn-au*pn)-p
        dQi[s2]=(qin-ai*qin)-qi[s2]; dQj[s2]=(qjn-ai*qjn)-qj[s2]
        np.add.at(P,uu[s2],dp)
        loss+=float(-np.log(s).sum())
    np.add.at(Q,ii,dQi); np.add.at(Q,jj,dQj)
    if (w0//W)%200==0: print(w0//W, time.time()-t0, flush=True)
print(json.dumps({'model':'Q stale within a window of %d triples (4 per lane group), P sequential per group, retirement order'%W,
  'loss_rel':abs(loss-lref)/lref,'P':bench.table_errors(P,Pr,P0),'Q':bench.table_errors(Q,Qr,Q0)},indent=1))
