"""Where the H-Codec-2.0 step's time goes in `qb_gemm`: one JSON document per run.

    python scripts/gemm_table.py --out DIR [--tag NAME] [--parts card,table,ksweep,smsweep,profile]

- card:    name, power limit and max SM clock (read-only nvidia-smi query).
- table:   every GEMM shape of the bench step (B = 64 x 10 s at 48 kHz, `mixed` policy) through `ops.gemm` with the epilogue
           `engine.cu` gives it; ms, issued TFLOP/s (split GEMMs count 3x), the kernel variant, and torch.matmul on fp16
           operands of the same M x N x K as the cuBLAS rate attainable on the same card (a speed yardstick, not a reference).
- ksweep:  pwconv1's shape at K in {768, 1536, 3072, 4608}, GELU -> fp16 hi and plain f32 out.  The slope of time over K is
           the main-loop rate, the intercept the per-tile fixed cost (epilogue and pipeline fill).
- smsweep: pwconv1 / pwconv2 at QB_GEMM_SMS = 132, 99, 66, each in its own process (the value is read once per process).
- profile: one `graphed('roundtrip')` replay at the bench shape under torch.profiler, total CUDA time per kernel name.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

M = 64 * 500                     # rows of the 50 Hz frame grid: B = 64 clips x 500 frames
C, I, IT = 1536, 4608, 4096      # model width, ConvNeXt hidden, transformer SwiGLU hidden


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clk = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(name=name, power_limit=power, clocks_max_sm=clk)


def timed(fn, min_s=0.5):
    """Mean ms per call over a window of at least min_s seconds of CUDA-event time, after a warm-up."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record(); torch.cuda.synchronize()
    reps = max(3, int(min_s * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def planes(shape, split, g, scale=1.0):
    from unified_audio_b200 import ops
    x = torch.randn(*shape, generator=g, device="cuda") * scale
    return ops.Planes.from_f32(x, split)


def case(name, *, m, n, k, split, taps=1, stride=1, batch=1, m_per_batch=None, a_rpb=None, bias=False, gamma=False,
         residual=False, inplace=False, act=0, act2=0, out="f32", out_ld=None, planes_pad=0):
    """One ops.gemm call built the way engine.cu builds it.  Returns (callable, issued FLOP, (M, N, K) for torch.matmul,
    the kernel variant qb_gemm picks).  inplace: the residual is the fp32 output itself; planes_pad: the planes are written
    at row offset planes_pad of (m_per_batch + 2 planes_pad)-row batches, the zero-padded input of the next conv."""
    from unified_audio_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    mpb = m_per_batch or m // batch
    rpb = a_rpb or mpb * stride + (taps - 1)
    rpb += (-rpb) % stride
    a = planes((batch * rpb, k), split, g)
    w = planes((n, taps * k), split, g, 1.0 / (taps * k) ** 0.5)
    n_out = n // 2 if act == ops.ACT_SWIGLU else n
    ld = out_ld or n_out
    kw = dict(a_batch=batch, a_rows_per_batch=rpb, a_ld=k, m_per_batch=mpb, taps=taps, stride=stride, act=act, act2=act2)
    if bias:
        kw["bias"] = torch.randn(n, generator=g, device="cuda")
    if gamma:
        kw["gamma"] = torch.randn(n, generator=g, device="cuda")
    if act == ops.ACT_SNAKE or act2 == ops.ACT_SNAKE:
        kw["act_param" if act == ops.ACT_SNAKE else "act2_param"] = torch.rand(n, generator=g, device="cuda") + 0.5
    keep = []
    if out in ("f32", "f32+planes"):
        o = torch.randn(batch * mpb, ld, generator=g, device="cuda")
        keep.append(o)
        kw["out_f32"] = ops.rowmap(o, ld, mpb, 0)
    if residual and inplace:
        kw["residual"] = kw["out_f32"]
    elif residual:
        r = torch.randn(batch * mpb, ld, generator=g, device="cuda")
        keep.append(r)
        kw["residual"] = ops.rowmap(r, ld, mpb, 0)
    if out in ("planes", "f32+planes"):
        kw["out_planes"] = ops.Planes.zeros((batch * (mpb + 2 * planes_pad), ld), split, "cuda")
        kw["out_planes_map"] = (ld, mpb + 2 * planes_pad, planes_pad)
    fn = lambda: ops.gemm(a, w, n, **kw)     # noqa: E731
    fn._keep = keep
    flop = 2.0 * batch * mpb * n * taps * k * (3 if split else 1)
    return fn, flop, (batch * mpb, n, taps * k), ops.gemm_kernel_name(mpb, n, split)


def shapes():
    """The bench step's GEMMs (engine.cu, `mixed` policy): name, calls per step, case kwargs."""
    from unified_audio_b200 import ops
    return [
        ("convnext.pwconv1", 56, dict(m=M, n=I, k=C, split=False, bias=True, act=ops.ACT_GELU, out="planes")),
        ("convnext.pwconv2", 56, dict(m=M, n=C, k=I, split=False, bias=True, gamma=True, residual=True)),
        ("tf.w_ih", 4, dict(m=M, n=4 * C, k=C, split=False, bias=True)),
        ("tf.qkv", 4, dict(m=M, n=3 * C, k=C, split=False, bias=True)),
        ("tf.o", 4, dict(m=M, n=C, k=C, split=False, residual=True)),
        ("tf.w13_swiglu", 4, dict(m=M, n=2 * IT, k=C, split=True, act=ops.ACT_SWIGLU, out="planes")),
        ("tf.w2", 4, dict(m=M, n=C, k=IT, split=True, residual=True)),
        ("resnet.conv_k3", 8, dict(m=M, n=C, k=C, split=True, taps=3, batch=64, bias=True, residual=True)),
    ] + sem_shapes() + [
        ("enc.out_conv_strided", 1, dict(m=64 * 125, n=1024, k=C, split=True, taps=9, stride=4, batch=64, bias=True)),
        ("dec.head", 1, dict(m=M, n=1922, k=C, split=True, bias=True, out_ld=1984)),
        ("stft.stage1_n128", 1, dict(m=M * 30, n=128, k=64, split=True)),
    ]


def sem_shapes():
    """encode_sem (engine.cu) at the bench shape: 768 -> 1536 channels, blocks at 500, 250 and 250 frames per clip with
    strides 2, 1, 2.  Every conv but the last writes fp16 hi + lo planes for the next one."""
    from unified_audio_b200 import ops
    B, Cs, ELU = 64, 1536, ops.ACT_ELU
    sem = dict(split=True, batch=64, n=Cs, k=Cs)
    planes = dict(out="f32+planes", planes_pad=1)
    rows = [("sem.s_conv_k3@500", 1, dict(sem, m=B * 500, k=768, taps=3, act2=ELU, **planes))]
    for t, blocks in ((500, 1), (250, 2)):
        rows += [(f"sem.conv_k3_elu@{t}", 2 * blocks, dict(sem, m=B * t, taps=3, act=ELU, out="planes")),
                 (f"sem.conv_1x1_res_elu@{t}", blocks, dict(sem, m=B * t, residual=True, inplace=True, act2=ELU, **planes)),
                 (f"sem.conv_1x1_res@{t}", blocks, dict(sem, m=B * t, residual=True, inplace=True, **planes))]
    for i, (t, s, act2) in enumerate(((500, 2, ELU), (250, 1, ELU), (250, 2, 0))):
        rows.append((f"sem.block{i}_conv_s{s}@{t}", 1, dict(sem, m=B * (t // s), taps=3, stride=s, bias=True, act2=act2, **planes)))
    rows.append(("sem.conv2@125", 1, dict(sem, m=B * 125, n=512, taps=3)))
    return rows


def matmul_rate(mnk):
    m, n, k = mnk
    a = torch.randn(m, k, device="cuda", dtype=torch.float16)
    b = torch.randn(k, n, device="cuda", dtype=torch.float16)
    ms = timed(lambda: torch.matmul(a, b))
    return dict(ms=ms, tflops=2.0 * m * n * k / ms / 1e9)


def part_table():
    rows = []
    for name, calls, kw in shapes():
        fn, flop, mnk, kern = case(name, **kw)
        ms = timed(fn)
        rows.append(dict(name=name, calls_per_step=calls, mnk=list(mnk), split=kw["split"], kernel=kern, m_per_batch=mnk[0] // kw.get("batch", 1), ms=ms,
                         tflops_issued=flop / ms / 1e9, ms_per_step=ms * calls, cublas_fp16=matmul_rate(mnk)))
        del fn
        torch.cuda.empty_cache()
    return rows


def part_ksweep():
    from unified_audio_b200 import ops
    out = []
    for epi, kw in (("gelu_hi", dict(bias=True, act=ops.ACT_GELU, out="planes")), ("f32", dict())):
        for k in (768, 1536, 3072, 4608):
            fn, flop, _, _ = case("ksweep", m=M, n=I, k=k, split=False, **kw)
            ms = timed(fn)
            out.append(dict(epilogue=epi, K=k, ms=ms, tflops=flop / ms / 1e9))
            del fn
    return out


def part_smsweep_child():
    fn1, f1, _, _ = case("pwconv1", **shapes()[0][2])
    fn2, f2, _, _ = case("pwconv2", **shapes()[1][2])
    sms = int(os.environ["QB_GEMM_SMS"])
    r = {}
    for nm, fn, f in (("pwconv1", fn1, f1), ("pwconv2", fn2, f2)):
        ms = timed(fn)
        r[nm] = dict(ms=ms, tflops=f / ms / 1e9, tflops_per_sm=f / ms / 1e9 / sms)
    return r


def part_smsweep():
    out = {}
    for sms in (132, 99, 66):
        env = dict(os.environ, QB_GEMM_SMS=str(sms))
        r = subprocess.run([sys.executable, __file__, "--child", "smsweep"], env=env, capture_output=True, text=True)
        out[str(sms)] = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else dict(error=r.stderr[-2000:])
    return out


def part_profile_child():
    import bench
    from torch.profiler import ProfilerActivity, profile
    cfg = bench.H2_FULL
    model = bench.build_codec(cfg, torch.device("cuda"), "mixed")
    wav_h, feat_h, _ = bench.synth_batch(cfg, 64, 10.0, 2000)
    graphed = model.graphed("roundtrip", wav_h.cuda(), feat_h.cuda())
    for _ in range(2):
        graphed()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        graphed()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            d = per.setdefault(ev.name, [0.0, 0])
            d[0] += ev.device_time_total / 1e3
            d[1] += 1
    total = sum(v[0] for v in per.values())
    rows = sorted(([k, v[0], v[1]] for k, v in per.items()), key=lambda r: -r[1])
    return dict(total_kernel_ms=total, kernels=[dict(name=n[:160], ms=t, calls=c, share=t / total) for n, t, c in rows[:40]])


def part_profile():
    r = subprocess.run([sys.executable, __file__, "--child", "profile"], capture_output=True, text=True)
    return json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else dict(error=r.stderr[-2000:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="directory the JSON document is written to")
    ap.add_argument("--tag", default="gemm_table")
    ap.add_argument("--parts", default="card,table,ksweep,smsweep,profile")
    ap.add_argument("--child", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_table.py measures on the GPU; none found"
    if args.child:
        print(json.dumps(part_smsweep_child() if args.child == "smsweep" else part_profile_child()))
        return
    if not args.out:
        ap.error("--out is required")
    doc = {}
    for part in args.parts.split(","):
        doc[part] = dict(card=card, table=part_table, ksweep=part_ksweep, smsweep=part_smsweep, profile=part_profile)[part]()
        if part == "table":
            doc["table_ms_per_step"] = sum(r["ms_per_step"] for r in doc[part])
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, args.tag + ".json")
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
    print(path)


if __name__ == "__main__":
    main()
