"""Host-side tile plans of the TMA-staged convolution kernel (no GPU): at the benchmark's shape, (B, T, H, W) =
(32, 32, 128, 128), the forward and backward passes of S3D send the same convolution launches to the TMA kernel as the
kernel with the shared-memory transpose epilogue did, and no launch gets fewer A-slab or weight slots or epilogue
staging buffers than it had then (recorded below)."""
import ctypes as C

import torch  # noqa: F401  (the dry-run plan is built over CPU tensors)

# launches the TMA kernel accepts, in plan order: (phase, shape, a_slots, b_slots, stage_bufs); b_slots = 0: resident
# weights
ACCEPTED = [
    ('fwd M=4194304 N=64 K=256 k=144 s=1 tr=0 C=16', 2, 0, 2),
    ('fwd M=2097152 N=64 K=448 k=711 s=2 tr=0 C=64', 2, 4, 2),
    ('fwd M=524288 N=64 K=64 k=111 s=1 tr=0 C=64', 4, 0, 2),
    ('fwd M=524288 N=192 K=576 k=133 s=1 tr=0 C=64', 2, 4, 2),
    ('fwd M=524288 N=192 K=576 k=311 s=1 tr=0 C=192', 2, 4, 2),
    ('fwd M=131072 N=112 K=192 k=111 s=1 tr=0 C=192', 2, 0, 2),
    ('fwd M=131072 N=128 K=384 k=311 s=1 tr=0 C=128', 2, 3, 2),
    ('fwd M=131072 N=64 K=192 k=111 s=1 tr=0 C=192', 4, 0, 2),
    ('fwd M=131072 N=32 K=192 k=111 s=1 tr=0 C=192', 4, 0, 2),
    ('fwd M=131072 N=160 K=256 k=111 s=1 tr=0 C=256', 2, 4, 2),
    ('fwd M=131072 N=192 K=1152 k=133 s=1 tr=0 C=128', 2, 4, 2),
    ('fwd M=131072 N=192 K=576 k=311 s=1 tr=0 C=192', 2, 4, 2),
    ('fwd M=131072 N=128 K=256 k=111 s=1 tr=0 C=256', 2, 0, 1),
    ('fwd M=131072 N=64 K=256 k=111 s=1 tr=0 C=256', 3, 0, 2),
    ('fwd M=16384 N=112 K=480 k=111 s=1 tr=0 C=480', 2, 3, 2),
    ('fwd M=16384 N=192 K=480 k=111 s=1 tr=0 C=480', 2, 4, 2),
    ('fwd M=16384 N=64 K=480 k=111 s=1 tr=0 C=480', 3, 4, 2),
    ('fwd M=16384 N=136 K=512 k=111 s=1 tr=0 C=512', 2, 4, 2),
    ('fwd M=16384 N=64 K=192 k=311 s=1 tr=0 C=64', 2, 4, 2),
    ('fwd M=16384 N=160 K=512 k=111 s=1 tr=0 C=512', 2, 4, 2),
    ('fwd M=16384 N=64 K=512 k=111 s=1 tr=0 C=512', 3, 4, 2),
    ('fwd M=16384 N=152 K=512 k=111 s=1 tr=0 C=512', 2, 4, 2),
    ('fwd M=16384 N=64 K=192 k=311 s=1 tr=0 C=64', 2, 4, 2),
    ('fwd M=16384 N=256 K=768 k=311 s=1 tr=0 C=256', 2, 3, 2),
    ('fwd M=16384 N=128 K=512 k=111 s=1 tr=0 C=512', 2, 3, 2),
    ('fwd M=16384 N=64 K=512 k=111 s=1 tr=0 C=512', 3, 4, 2),
    ('fwd M=16384 N=176 K=512 k=111 s=1 tr=0 C=512', 2, 4, 2),
    ('fwd M=16384 N=64 K=192 k=311 s=1 tr=0 C=64', 2, 4, 2),
    ('fwd M=16384 N=112 K=512 k=111 s=1 tr=0 C=512', 2, 3, 2),
    ('fwd M=16384 N=64 K=512 k=111 s=1 tr=0 C=512', 3, 4, 2),
    ('fwd M=16384 N=192 K=528 k=111 s=1 tr=0 C=528', 2, 4, 2),
    ('fwd M=16384 N=128 K=384 k=311 s=1 tr=0 C=128', 2, 3, 2),
    ('fwd M=16384 N=320 K=960 k=311 s=1 tr=0 C=320', 2, 3, 2),
    ('fwd M=16384 N=256 K=528 k=111 s=1 tr=0 C=528', 2, 3, 2),
    ('fwd M=16384 N=128 K=528 k=111 s=1 tr=0 C=528', 2, 3, 2),
    ('fwd M=2048 N=192 K=832 k=111 s=1 tr=0 C=832', 2, 4, 2),
    ('fwd M=2048 N=256 K=832 k=111 s=1 tr=0 C=832', 2, 3, 2),
    ('fwd M=2048 N=128 K=832 k=111 s=1 tr=0 C=832', 2, 3, 2),
    ('fwd M=2048 N=240 K=832 k=111 s=1 tr=0 C=832', 2, 3, 2),
    ('fwd M=2048 N=384 K=832 k=111 s=1 tr=0 C=832', 2, 3, 2),
    ('fwd M=2048 N=128 K=832 k=111 s=1 tr=0 C=832', 2, 3, 2),
    ('fwd M=32 N=1024 K=1024 k=111 s=1 tr=0 C=1024', 2, 3, 2),
    ('fwd M=32 N=128 K=1024 k=111 s=1 tr=0 C=1024', 2, 3, 2),
    ('bwd M=32 N=1024 K=128 k=111 s=1 tr=1 C=128', 2, 3, 2),
    ('bwd M=32 N=1024 K=1024 k=111 s=1 tr=1 C=1024', 2, 3, 2),
    ('bwd M=2048 N=832 K=384 k=111 s=1 tr=1 C=384', 2, 3, 2),
    ('bwd M=2048 N=832 K=128 k=111 s=1 tr=1 C=128', 2, 3, 2),
    ('bwd M=2048 N=832 K=240 k=111 s=1 tr=1 C=240', 2, 3, 2),
    ('bwd M=2048 N=832 K=256 k=111 s=1 tr=1 C=256', 2, 3, 2),
    ('bwd M=2048 N=832 K=128 k=111 s=1 tr=1 C=128', 2, 3, 2),
    ('bwd M=2048 N=832 K=192 k=111 s=1 tr=1 C=192', 2, 3, 2),
    ('bwd M=16384 N=128 K=384 k=311 s=1 tr=1 C=128', 2, 3, 2),
    ('bwd M=16384 N=320 K=960 k=311 s=1 tr=1 C=320', 2, 3, 2),
    ('bwd M=16384 N=528 K=256 k=111 s=1 tr=1 C=256', 2, 3, 2),
    ('bwd M=16384 N=528 K=128 k=111 s=1 tr=1 C=128', 2, 3, 2),
    ('bwd M=16384 N=528 K=192 k=111 s=1 tr=1 C=192', 2, 3, 2),
    ('bwd M=16384 N=64 K=192 k=311 s=1 tr=1 C=64', 2, 4, 2),
    ('bwd M=16384 N=512 K=112 k=111 s=1 tr=1 C=112', 2, 3, 2),
    ('bwd M=16384 N=512 K=64 k=111 s=1 tr=1 C=64', 2, 3, 2),
    ('bwd M=16384 N=512 K=176 k=111 s=1 tr=1 C=176', 2, 3, 2),
    ('bwd M=16384 N=64 K=192 k=311 s=1 tr=1 C=64', 2, 4, 2),
    ('bwd M=16384 N=256 K=768 k=311 s=1 tr=1 C=256', 2, 3, 2),
    ('bwd M=16384 N=512 K=128 k=111 s=1 tr=1 C=128', 2, 3, 2),
    ('bwd M=16384 N=512 K=64 k=111 s=1 tr=1 C=64', 2, 3, 2),
    ('bwd M=16384 N=512 K=152 k=111 s=1 tr=1 C=152', 2, 3, 2),
    ('bwd M=16384 N=64 K=192 k=311 s=1 tr=1 C=64', 2, 4, 2),
    ('bwd M=16384 N=512 K=160 k=111 s=1 tr=1 C=160', 2, 3, 2),
    ('bwd M=16384 N=512 K=64 k=111 s=1 tr=1 C=64', 2, 3, 2),
    ('bwd M=16384 N=512 K=136 k=111 s=1 tr=1 C=136', 2, 3, 2),
    ('bwd M=16384 N=480 K=192 k=111 s=1 tr=1 C=192', 2, 3, 2),
    ('bwd M=16384 N=480 K=64 k=111 s=1 tr=1 C=64', 2, 3, 2),
    ('bwd M=16384 N=480 K=112 k=111 s=1 tr=1 C=112', 2, 3, 2),
    ('bwd M=131072 N=192 K=576 k=311 s=1 tr=1 C=192', 2, 4, 2),
    ('bwd M=131072 N=256 K=128 k=111 s=1 tr=1 C=128', 2, 3, 2),
    ('bwd M=131072 N=256 K=64 k=111 s=1 tr=1 C=64', 2, 3, 2),
    ('bwd M=131072 N=128 K=1728 k=133 s=1 tr=1 C=192', 2, 3, 2),
    ('bwd M=131072 N=256 K=160 k=111 s=1 tr=1 C=160', 2, 3, 2),
    ('bwd M=131072 N=128 K=384 k=311 s=1 tr=1 C=128', 2, 3, 2),
    ('bwd M=131072 N=192 K=64 k=111 s=1 tr=1 C=64', 2, 4, 2),
    ('bwd M=131072 N=192 K=32 k=111 s=1 tr=1 C=32', 2, 4, 2),
    ('bwd M=131072 N=96 K=1152 k=133 s=1 tr=1 C=128', 2, 4, 2),
    ('bwd M=131072 N=192 K=112 k=111 s=1 tr=1 C=112', 2, 4, 2),
    ('bwd M=524288 N=192 K=576 k=311 s=1 tr=1 C=192', 2, 4, 2),
    ('bwd M=524288 N=64 K=1728 k=133 s=1 tr=1 C=192', 3, 4, 2),
    ('bwd M=524288 N=64 K=64 k=111 s=1 tr=1 C=64', 4, 0, 2),
    ('bwd M=4194304 N=64 K=448 k=711 s=2 tr=1 C=64', 2, 4, 2),
]
N_LAUNCHES = 139   # coclr_conv_igemm launches of one forward + backward pass; the others run on the gather kernel


def _key(phase, o):
    return "%s M=%d N=%d K=%d k=%d%d%d s=%d tr=%d C=%d" % (phase, o.B * o.Td * o.Hd * o.Wd, o.N, o.Kreal, o.g.kt,
                                                         o.g.kh, o.g.kw, o.g.st, o.g.transposed, o.src.C)


def test_tma_plans_of_the_benchmark_shape():
    from coclr_b200 import lib as L, engine as E
    from coclr_b200.s3d_spec import s3d_stages
    lib = L.load()
    L.DRY_RUN = True
    try:
        g = E.Graph(s3d_stages(3), 3, head_dim=128, bb_prefix="0.")
        st = E.ParamStore(g, "cpu")
        eng = E.EncoderEngine(st, g, "parity")
        p = eng.plan(32, 32, 128, 128, True, True)
        info = (C.c_int * 8)()
        seen, accepted = 0, []
        for phase, lst in (("fwd", p.fwd), ("bwd", p.bwd)):
            for fn, a in lst:
                if fn.__name__ != "coclr_conv_igemm":
                    continue
                seen += 1
                if lib.coclr_conv_tma_plan(a[0], info) == 1:
                    accepted.append((_key(phase, a[0]._obj), info[0], info[1], info[2], info[3]))
        assert seen == N_LAUNCHES
        assert [k for k, *_ in accepted] == [k for k, *_ in ACCEPTED]
        for (key, a_slots, b_slots, resident, stage_bufs), (_, a_was, b_was, bufs_was) in zip(accepted, ACCEPTED):
            assert stage_bufs >= bufs_was, key
            assert a_slots >= a_was, (key, a_slots, a_was)
            assert (b_slots == 0) == bool(resident), key
            assert b_slots >= b_was if b_was else resident, (key, b_slots, b_was)
    finally:
        L.DRY_RUN = False
