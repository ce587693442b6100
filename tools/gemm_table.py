"""Aggregate a NRW_GEMM_TIMING_DUMP csv: per GEMM configuration count, time, MMA rate and HBM rate.  A paired backward launch
(mn 3) carries its weight gradient's shape as well (the `dW M x N x K/ks` column); its MMA rate counts both GEMMs."""
import sys, collections
rows = collections.OrderedDict()
for l in open(sys.argv[1]):
    f = l.strip().split(",")
    M, N, K, P, mn, ks, epi, by, ms = f[:9]
    dw = tuple(int(x) for x in f[9:13]) if len(f) >= 13 else None
    k = (int(M), int(N), int(K), int(P), int(mn), int(ks), int(epi), dw)
    r = rows.setdefault(k, [0, 0.0, float(by)])
    r[0] += 1; r[1] += float(ms)
steps = float(sys.argv[2]) if len(sys.argv) > 2 else 1.0
tot = sum(r[1] for r in rows.values())
print(f"total {tot/steps:.2f} ms/step in {sum(r[0] for r in rows.values())/steps:.0f} launches")
print("     M     N     K P mn ks  epi |   n/step  ms/step   us/launch  MMA TF/s  GB/s(alg) | paired dW M x N x K/ks")
for k, r in sorted(rows.items(), key=lambda kv: -kv[1][1]):
    M, N, K, P, mn, ks, epi, dw = k
    us = r[1] / r[0] * 1e3
    npr = {1: 1, 2: 3, 3: 6}[P]
    flop = 2.0 * M * N * K * npr + (2.0 * dw[0] * dw[1] * dw[2] if dw else 0.0)
    pair = f" | {dw[0]} x {dw[1]} x {dw[2]}/{dw[3]}" if dw else ""
    print(f"{M:7d} {N:5d} {K:6d} {P} {mn:2d} {ks:3d} {epi:4d} | {r[0]/steps:7.1f} {r[1]/steps:8.2f} {us:10.1f} {flop/us/1e6:9.0f} {r[2]/us/1e3:9.0f}{pair}")
