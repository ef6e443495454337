"""Small driver for compute-sanitizer (memcheck / racecheck): every kernel once on small inputs."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import bodywork_mlops_demo_b200 as b2
from oracle import ols_oracle as orc
which = sys.argv[1] if len(sys.argv) > 1 else "all"
ctx = b2.Context(0)
X, y = orc.generate_dataset(4096 + 37, 128, seed=1, dtype=np.float32)
mask = (np.arange(len(y)) % 5 != 0).astype(np.uint8)
Xd, yd, md = ctx.to_device(X), ctx.to_device(y), ctx.to_device(mask)
if which in ("all", "simt"):
    ctx.set_kernel(b2.KERNEL_SIMT); ctx.gram_reset(128); ctx.gram_accumulate(Xd, yd, md, 1)
    print("simt n", ctx.gram_export()[128, 128])
if which in ("all", "tc"):
    ctx.set_kernel(b2.KERNEL_TCGEN05); ctx.set_drain_rows(1024); ctx.gram_reset(128); ctx.gram_accumulate(Xd, yd, md, 1)
    print("tc n", ctx.gram_export()[128, 128])
if which in ("all", "solve"):
    ctx.gram_import(orc.gram_stats(X, y))
    c, b = ctx.solve(); c2, b2_, s, r = ctx.solve_spectral()
    print("solve", c[:2], r)
    X3, y3 = orc.generate_dataset(500, 33, seed=2)
    ctx.gram_import(orc.gram_stats(X3, y3)); print("solve33", ctx.solve()[0][:2], ctx.solve_spectral()[3])
if which in ("all", "score"):
    yh, st = ctx.score(Xd, np.full(128, 0.5), 1.0, y=yd, row_mask=md, mask_keep=0)
    print("score", st[5])
    Xs, ys = ctx.synth(1000, 128, seed=3); print("synth", float(Xs.to_host().mean()))
if which in ("all", "narrow"):
    # narrow-row Gram (one lane per row, two lanes per row, two rows per pair) and narrow-row scoring, with a mask
    for d in (1, 3, 8, 12, 16):
        Xn, yn = orc.generate_dataset(9000 + d, d, seed=10 + d, dtype=np.float32)
        mn = (np.arange(len(yn)) % 4 != 0).astype(np.uint8)
        Xnd, ynd, mnd = ctx.to_device(Xn), ctx.to_device(yn), ctx.to_device(mn)
        ctx.set_kernel(b2.KERNEL_NARROW); ctx.gram_reset(d); ctx.gram_accumulate(Xnd, ynd, mnd, 1)
        S = ctx.gram_export()
        _, st = ctx.score(Xnd, np.full(d, 0.5), 1.0, y=ynd, row_mask=mnd, mask_keep=0)
        print("narrow", d, S[d, d], st[5])
        for a in (Xnd, ynd, mnd): a.free()
    ctx.set_kernel(b2.KERNEL_AUTO)
if which in ("all", "packed"):
    # packed super-rows on the tensor-core path (pack = 5 with the 2-D mask view, pack = 3) and the streaming scorer
    for d in (24, 40, 64):
        Xp, yp = orc.generate_dataset(6000 + d, d, seed=20 + d, dtype=np.float32)
        mp = (np.arange(len(yp)) % 3 != 0).astype(np.uint8)
        Xpd, ypd, mpd = ctx.to_device(Xp), ctx.to_device(yp), ctx.to_device(mp)
        ctx.set_kernel(b2.KERNEL_TCGEN05); ctx.gram_reset(d); ctx.gram_accumulate(Xpd, ypd, mpd, 1)
        S = ctx.gram_export()
        _, st = ctx.score(Xpd, np.full(d, 0.5), 1.0, y=ypd, row_mask=mpd, mask_keep=0)
        print("packed", d, S[d, d], st[5])
        for a in (Xpd, ypd, mpd): a.free()
    ctx.set_kernel(b2.KERNEL_AUTO)
if which in ("all", "fit"):
    # round 2: the one-call fit (shift sample, Gram, cooperative finalize, LDL^T solve), the eigenvalue kernel, the
    # metrics-only narrow scorer, float64 metrics, the device tranche generator
    ctx.set_kernel(b2.KERNEL_TCGEN05); ctx.set_drain_rows(1024)
    c, b = ctx.fit(Xd, yd, md, 1)
    sing, rank, rows = ctx.solve_eigvals()
    print("fit", c[:2], rank, rows)
    X3, y3 = orc.generate_dataset(700, 33, seed=2, dtype=np.float32)
    ctx.set_kernel(b2.KERNEL_AUTO)
    c3, b3 = ctx.fit(X3, y3); print("fit33 host rows", c3[:2], ctx.solve_eigvals()[1])
    for d in (1, 2, 8):
        Xn, yn = orc.generate_dataset(20000 + d, d, seed=30 + d, dtype=np.float32)
        Xnd, ynd = ctx.to_device(Xn), ctx.to_device(yn)
        _, st = ctx.score(Xnd, np.full(d, 0.5), 1.0, y=ynd, want_yhat=False)
        print("score plain", d, st[5]); Xnd.free(); ynd.free()
    print("metrics", ctx.metrics(y.astype(np.float64), y.astype(np.float64) * 1.01)[5])
    Xt, yt, kept = ctx.synth_tranche(5000, 7, seed=5); print("tranche", kept); Xt.free(); yt.free()
if which in ("all", "b16"):
    # bf16-stored rows, D = 128: the raw swizzled tile as the wgmma B operand, one merged accumulator, both operand
    # modes, with a mask and a ragged last tile, short drain interval
    Xb = b2.native.to_bf16_bits(X)
    Xbd = ctx.to_device(Xb, "bf16")
    ctx.set_kernel(b2.KERNEL_TCGEN05); ctx.set_drain_rows(1024)
    for prec in (b2.PRECISION_SPLIT, b2.PRECISION_BF16):
        ctx.set_precision(prec)
        ctx.gram_reset(128); ctx.gram_accumulate(Xbd, yd, md, 1)
        print("b16 masked n", ctx.gram_export()[128, 128])
        c, b = ctx.fit(Xbd, yd)
        print("b16 fit", c[:2])
    ctx.set_precision(b2.PRECISION_SPLIT); ctx.set_drain_rows(8192); ctx.set_kernel(b2.KERNEL_AUTO)
    Xbd.free()
if which in ("all", "xchg"):
    # peer-memory exchange between two contexts on this device: finalize-kernel scatter + solve-kernel gather, and the
    # stand-alone scatter / gather kernels
    import threading
    cs = [ctx, b2.Context(0)]
    b2.Context.comm_p2p_attach_local(cs)
    half = len(y) // 2
    sh = [(cs[0].to_device(X[:half]), cs[0].to_device(y[:half])), (cs[1].to_device(X[half:]), cs[1].to_device(y[half:]))]
    out = [None, None]
    for mode in ("fused", "standalone"):
        def work(i):
            c = cs[i]
            c.set_kernel(b2.KERNEL_TCGEN05)
            if mode == "fused":
                out[i] = c.fit(sh[i][0], sh[i][1])
            else:
                c.gram_reset(128); c.gram_accumulate(sh[i][0], sh[i][1]); c.gram_allreduce(); out[i] = c.solve()
        ts = [threading.Thread(target=work, args=(i,)) for i in range(2)]
        [t.start() for t in ts]; [t.join() for t in ts]
        print("xchg", mode, out[0][0][:2], bool(np.array_equal(out[0][0], out[1][0])), cs[0].gram_export()[128, 128])
    for c in cs: c.comm_p2p_detach()
    cs[1].close()
print("done")
