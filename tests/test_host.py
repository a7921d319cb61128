"""CPU-only checks: module ABI vs the reference, C-ABI symbols, loud failure without a GPU."""
import ast
import ctypes
import glob
import json
import os
import re
import warnings

import numpy as np
import pytest
import torch

from conftest import ROOT
from melgan_multi_b200 import engine, synth
from kernel_model import NORMS, check_grad_digest, mel_option_cases, train_case

warnings.filterwarnings("ignore")


@pytest.fixture(scope="module")
def abi():
    with open(os.path.join(ROOT, "tests", "golden", "module_abi.json")) as f:
        return json.load(f)


def test_generator_module_abi_matches_reference(abi):
    from melgan_multi_b200 import models
    g = models.Generator()
    got = [[k, list(v.shape)] for k, v in g.state_dict().items()]
    assert got == abi["Generator"]["state_dict"]
    assert [n for n, _ in g.named_parameters()] == abi["Generator"]["parameters"]
    assert sum(p.numel() for p in g.parameters()) == 4524290


def test_msd_module_abi_matches_reference(abi):
    from melgan_multi_b200 import models
    d = models.MultiScaleDiscriminator()
    got = [[k, list(v.shape)] for k, v in d.state_dict().items()]
    assert got == abi["MultiScaleDiscriminator"]["state_dict"]
    assert [n for n, _ in d.named_parameters()] == abi["MultiScaleDiscriminator"]["parameters"]
    assert sum(p.numel() for p in d.parameters()) == 16924086


def test_synth_state_matches_module_abi(abi):
    gs = synth.generator_state(1)
    assert [[k, list(v.shape)] for k, v in gs.items()] == abi["Generator"]["state_dict"]
    ds = synth.discriminator_state(1)
    assert [[k, list(v.shape)] for k, v in ds.items()] == abi["MultiScaleDiscriminator"]["state_dict"]
    # seeded and reproducible
    assert np.array_equal(gs["ups.2.weight_v"], synth.generator_state(1)["ups.2.weight_v"])


def test_cabi_library_exports_every_declared_symbol():
    """Every function declared in include/melgan_b200.h must be exported by the built library."""
    hdr = open(os.path.join(ROOT, "include", "melgan_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = re.findall(r"\b(mg_[a-z0-9_]+)\s*\(", hdr)
    assert len(set(names)) >= 14
    lib = ctypes.CDLL(engine.LIB_PATH)
    for n in set(names):
        assert hasattr(lib, n), "missing export %s" % n
    assert engine.lib().mg_abi_version() == 2
    fp32_blob = (4524290 - 4353) * 4
    tc_blob = 6 * 12 * (256 * 256 + 128 * 128 + 64 * 64 + 32 * 32)  # split-bf16 copy of the 24 ResBlock convs
    tc_blob += 4 * (512 * 256 * 16 + 256 * 128 * 16 + 128 * 64 * 4 + 64 * 32 * 4)  # ... and of the 4 ConvTranspose1d
    tc_blob += 4 * 80 * 512 * 7  # ... and of conv_pre
    tc_blob += 4 * (128 * 64 * 4 + 64 * 32 * 4)  # ... and of the stride-2 ConvTs again, in the fused stage kernels' layout
    assert engine.lib().mg_gen_packed_bytes() == (fp32_blob + 255) // 256 * 256 + tc_blob
    assert engine.lib().mg_gen_workspace_bytes(64, 32) == 64 * 32 * (18944 + 2 * 8192) * 4 + 256
    assert engine.lib().mg_gen_workspace_bytes(0, 32) == 0


def test_generator_refuses_cpu_tensors():
    from melgan_multi_b200 import models
    g = models.Generator()
    with pytest.raises(engine.EngineError):
        g(torch.zeros(1, 80, 4))


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_engine_fails_loudly_without_gpu():
    with pytest.raises(engine.EngineError):
        engine.GeneratorHost(1, 4)
    assert "CUDA" in engine.lib().mg_last_error_string().decode() or "cuda" in engine.lib().mg_last_error_string().decode()


def test_torch_restatement_used_for_backward_matches_golden(golden):
    """Generator._torch_forward (the stock-op graph autograd differentiates) == reference output."""
    import cases
    from melgan_multi_b200 import models
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    vs, gs_, bs = g._param_triplets()
    leaves = []
    for v, gg, b in zip(vs, gs_, bs):
        leaves += [v, gg, b]
    case = cases.GEN_CASES[1]
    with torch.no_grad():
        y = g._torch_forward(torch.from_numpy(synth.mel_input(*case)), leaves).numpy()
    ref = golden[cases.gen_key(*case)]
    assert np.abs(y - ref).max() <= 2e-5 * np.abs(ref).max()


def ref_feature_loss(fmap_r, fmap_g):
    """The reference's formulas (models.py:138-167) in plain torch: the CPU side of the loss tests (the product's loss
    functions are CUDA-only)."""
    return sum((r - g).abs().mean() for a, b in zip(fmap_r, fmap_g) for r, g in zip(a, b)) * 10


def ref_generator_loss(dg):
    return sum(((1 - g) ** 2).mean() for g in dg)


def ref_discriminator_loss(dr, dg):
    r = [((1 - x) ** 2).mean() for x in dr]
    g = [(x ** 2).mean() for x in dg]
    return sum(r) + sum(g), [v.item() for v in r], [v.item() for v in g]


def test_losses_match_reference_values(golden):
    """The stock-op graph that autograd differentiates (MultiScaleDiscriminator._torch_forward, CPU) + the reference's loss
    formulas reproduce the reference's loss values."""
    import cases
    from melgan_multi_b200 import models
    B, L, seed = cases.MSD_CASES[1]
    d = models.MultiScaleDiscriminator()
    d.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
    vs, gs_, bs = d._param_triplets()
    leaves = []
    for v, g, b in zip(vs, gs_, bs):
        leaves += [v, g, b]
    y2 = torch.cat([torch.from_numpy(synth.audio_input(B, L, seed)), torch.from_numpy(synth.audio_input(B, L, seed + 7))])
    with torch.no_grad():
        outs = d._torch_forward(y2, leaves)
    fm = [outs[7 * s:7 * s + 7] for s in range(3)]
    frs, fgs = [[f[:B] for f in sc] for sc in fm], [[f[B:] for f in sc] for sc in fm]
    rs, gs = [sc[6][:B].flatten(1) for sc in fm], [sc[6][B:].flatten(1) for sc in fm]
    tag = "msd_B%d_L%d_s%d" % (B, L, seed)
    assert abs(ref_feature_loss(frs, fgs).item() - float(golden[tag + "_feature_loss"])) < 1e-4
    assert abs(ref_generator_loss(gs).item() - float(golden[tag + "_generator_loss"])) < 1e-5
    dl, rl, gl = ref_discriminator_loss(rs, gs)
    with pytest.raises(engine.EngineError):  # the product's loss functions refuse CPU tensors, like the modules
        models.feature_loss(frs, fgs)
    np.testing.assert_allclose([dl.item()] + rl + gl, golden[tag + "_discriminator_loss"], rtol=1e-4, atol=1e-6)


def test_discriminators_refuse_cpu_tensors():
    from melgan_multi_b200 import models
    d = models.MultiScaleDiscriminator()
    with pytest.raises(engine.EngineError):
        d(torch.zeros(1, 1, 64), torch.zeros(1, 1, 64))
    with pytest.raises(engine.EngineError):
        d.discriminators[0](torch.zeros(1, 1, 64))


@pytest.mark.parametrize("make", [lambda ps: torch.optim.Adam(ps, fused=True), lambda ps: torch.optim.AdamW(ps, fused=True),
                                  lambda ps: torch.optim.SGD(ps, lr=0.1, fused=True)], ids=["Adam", "AdamW", "SGD"])
def test_fused_optimizer_steps_bump_the_versions_the_packed_weights_are_keyed_on(make):
    """torch's fused optimizer steps leave the parameters' version counters as they were; once models is imported,
    a step bumps those of every parameter it updated, as the for-loop and foreach steps do."""
    from melgan_multi_b200 import models  # noqa: F401 (registers the step hook)
    p, idle = torch.nn.Parameter(torch.randn(5)), torch.nn.Parameter(torch.randn(3))
    p.grad = torch.randn(5)
    opt = make([p, idle])
    v0 = p._version
    opt.step()
    assert p._version > v0 and idle._version == 0


def test_compiled_fused_optimizer_step_bumps_the_versions():
    from melgan_multi_b200 import models  # noqa: F401 (registers the step hook)
    p = torch.nn.Parameter(torch.randn(5))
    p.grad = torch.randn(5)
    opt = torch.optim.Adam([p], fused=True)
    step = torch.compile(lambda: opt.step())
    w0, v0 = p.detach().clone(), p._version
    step()
    assert not torch.equal(p.detach(), w0) and p._version > v0


def test_pack_key_sees_a_new_storage_at_the_packed_address():
    """p.data = t keeps p's version counter, and the caching allocator may hand t the address of the storage the last
    pack read once that storage is freed: (data_ptr, _version) then recurs, but the freed storage's weak reference has
    expired."""
    from melgan_multi_b200 import models
    ps = [torch.nn.Parameter(torch.randn(4)) for _ in range(3)]
    key = models._PackKey(ps)
    assert key.matches(ps)
    ps[1].data = torch.randn(4)  # the packed storage of ps[1] is freed here
    assert not key.matches(ps)
    key.key = tuple((t.data_ptr(), t._version) for t in ps)  # as if the new storage had landed at the packed address
    assert not key.matches(ps)
    assert models._PackKey(ps).matches(ps)


def test_repack_reaches_every_packed_module_inside():
    from melgan_multi_b200 import models
    msd = models.MultiScaleDiscriminator()
    for m in [msd] + list(msd.discriminators):
        m._packed_key = ("stale",)
    msd.repack()
    assert all(m._packed_key is None for m in [msd] + list(msd.discriminators))
    d = msd.discriminators[1]
    d._packed_key = msd._packed_key = ("stale",)
    d.repack()
    assert d._packed_key is None and msd._packed_key == ("stale",)


def test_simt_test_library_is_separate_from_the_product():
    """The first-generation fp32 SIMT generator is test infrastructure: it lives in its own library, and the product
    library neither exports nor contains it."""
    from melgan_multi_b200 import build
    prod = ctypes.CDLL(engine.LIB_PATH)
    assert not hasattr(prod, "mg_simt_gen_forward")
    assert os.path.exists(build.TEST_LIB) and hasattr(ctypes.CDLL(build.TEST_LIB), "mg_simt_gen_forward")
    for f in os.listdir(os.path.join(ROOT, "melgan_multi_b200")):
        if f.endswith(".py") and f != "build.py":
            assert "simt_test" not in open(os.path.join(ROOT, "melgan_multi_b200", f)).read(), f


def test_cabi_argument_errors_are_reported_not_thrown():
    """Error behaviour of the C ABI that needs no GPU: negative return code + message, never an exception or exit."""
    L = engine.lib()
    lens = (ctypes.c_int * 21)()
    assert L.mg_msd_lengths(0, lens) == -1 and b"mg_msd_lengths" in L.mg_last_error_string()
    assert L.mg_msd_lengths(8192, lens) == 0
    assert [lens[i] for i in range(7)] == [8192, 2048, 512, 128, 128, 128, 128]
    assert [lens[7 + i] for i in range(7)] == [4097, 1025, 257, 65, 65, 65, 65]
    assert [lens[14 + i] for i in range(7)] == [1025, 257, 65, 17, 17, 17, 17]
    assert engine.msd_lengths(1031)[2][6] >= 1
    # null / bad-shape arguments of the device-pointer entry points are rejected before any CUDA call
    assert L.mg_gen_forward(None, None, None, 1, 1, None, 0, None) == -1
    assert L.mg_gen_forward(ctypes.c_void_p(256), ctypes.c_void_p(256), ctypes.c_void_p(256), 0, 4,
                            ctypes.c_void_p(256), 1 << 30, None) == -1
    assert b"B >= 1" in L.mg_last_error_string()
    assert L.mg_gen_forward(ctypes.c_void_p(256), ctypes.c_void_p(256), ctypes.c_void_p(256), 1, 4,
                            ctypes.c_void_p(256), 16, None) == -4  # MG_ERR_WORKSPACE_TOO_SMALL
    assert L.mg_gen_kernel_name(0) == b"conv_pre" and L.mg_gen_kernel_name(99) == b""
    assert L.mg_gen_forward_launches() == 8 and L.mg_gen_kernel_name(7) == b"up3+res3+post" and L.mg_gen_kernel_name(2) == b"res0"
    assert L.mg_gen_set_pipeline(10) == 0 and L.mg_gen_forward_launches() == 7 and L.mg_gen_kernel_name(6) == b"res3+post"
    assert L.mg_gen_kernel_name(2) == b"res0+up1"
    assert L.mg_gen_set_pipeline(14) == 0 and L.mg_gen_forward_launches() == 6 and L.mg_gen_kernel_name(3) == b"res1+up2"
    assert L.mg_gen_set_pipeline(99) == -1 and L.mg_gen_set_pipeline(-1) == 0 and L.mg_gen_forward_launches() == 8
    assert L.mg_gen_resup(p0 := ctypes.c_void_p(256), 3, p0, ctypes.c_void_p(512), 1, 4, None) == -1  # stages 0..2 only
    # batch slices: config 2 runs as 4 chains, small or single-item batches as one
    assert [L.mg_gen_forward_slices(b, t) for b, t in ((64, 32), (40, 32), (16, 32), (1, 1000), (0, 5))] == [4, 2, 1, 1, 1]
    # the training-side entry points validate before touching the device too
    p = ctypes.c_void_p(256)
    assert L.mg_gen_upres(p, 1, p, ctypes.c_void_p(512), 1, 4, None) == -1  # only stages 2 and 3 are stride-2
    n1 = (ctypes.c_longlong * 1)(16)
    m1 = (ctypes.c_int * 1)(7)
    a1 = (ctypes.c_void_p * 1)(256)
    assert L.mg_loss_workspace_bytes(n1, 1) == 4 and L.mg_loss_workspace_bytes(None, 1) == 0
    assert L.mg_loss_forward(a1, a1, n1, m1, 1, p, p, 4, None) == -1 and b"bad row" in L.mg_last_error_string()  # mode 7
    assert L.mg_loss_forward(a1, a1, n1, m1, 0, p, p, 4, None) == -1 and L.mg_loss_backward(a1, a1, n1, m1, 1, None, a1, a1, None) == -1
    assert L.mg_msd_grouped_backward_workspace_bytes(5, 2, 64) == 0 and L.mg_msd_grouped_backward_workspace_bytes(1, 2, 64) > 0
    assert L.mg_msd_grouped_backward(p, 0, 1, p, p, p, p, p, p, 1 << 30, 2, 1024, 999, None) == -1
    assert b"does not follow" in L.mg_last_error_string()  # Lout must be the conv's output length for Lin
    assert L.mg_msd_grouped_backward(p, 0, 1, p, p, p, p, p, p, 8, 2, 1024, 256, None) == -4  # workspace too small
    assert L.mg_msd_wn_backward(None, None, None, None, None, None) == -1 and L.mg_lrelu_backward(None, None, None, None, 4, None) == -1
    assert L.mg_gen_conv_pre(None, None, None, 1, 1, None) == -1 and L.mg_gen_resblock_post(p, p, p, 0, 4, None) == -1
    assert L.mg_disc_packed_bytes() * 3 == L.mg_msd_packed_bytes()
    assert L.mg_disc_pack(None, None, None, None, None) == -1 and L.mg_disc_forward(p, p, 1, 0, p, p, None) == -1
    assert L.mg_adam_chunk() == 4096 and L.mg_adam_step(None, None, None, None, None, None, 1, 1, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, None) == -1
    # round-2 backward entry points of the discriminators: conv_post1 dgrad / wgrad, conv_pre / conv_post2, the one-call chain
    assert L.mg_msd_post1_dgrad(p, 3, p, ctypes.c_void_p(512), 2, 8, p, None) == -1  # scale 0..2
    assert L.mg_msd_post1_dgrad(p, 0, p, p, 2, 8, p, None) == -1                     # dz and dx must differ
    assert L.mg_msd_post1_wgrad(p, p, None, p, 2, 8, p, None) == -1
    assert L.mg_msd_edge_backward_workspace_bytes(0, 2, 1024) == 2 * 2 * 256 * 4 and L.mg_msd_edge_backward_workspace_bytes(6, 2, 64) == 0
    assert L.mg_msd_edge_backward(p, 0, 3, p, p, p, p, p, p, 1 << 20, 2, 64, None) == -1 and b"layer is 0" in L.mg_last_error_string()
    assert L.mg_msd_edge_backward(p, 0, 0, p, p, p, p, p, p, 16, 2, 1024, None) == -4  # conv_pre needs its workspace
    big, small = L.mg_msd_scale_backward_workspace_bytes(32, 8192), L.mg_msd_scale_backward_workspace_bytes(2, 1024)
    assert big > small > 0 and L.mg_msd_scale_backward_workspace_bytes(0, 64) == 0
    assert big >= 3 * 32 * 16 * 8192 * 4  # dz + two alternating dx buffers of the largest activation
    seven = (ctypes.c_void_p * 7)(*([256] * 7))
    none7 = (ctypes.c_void_p * 7)()
    assert L.mg_msd_scale_backward(p, 0, p, none7, seven, None, seven, seven, None, p, big, 2, 1024, p, None) == -1
    assert b"fmap[0]" in L.mg_last_error_string()
    assert L.mg_msd_scale_backward(p, 0, p, seven, seven, None, seven, seven, None, p, 16, 2, 1024, p, None) == -4


def test_backward_restatement_matches_reference_gradients():
    """The stock-op graphs the autograd path differentiates (Generator._torch_forward / MultiScaleDiscriminator.
    _torch_forward + the reference's loss formulas), run on CPU through one train.py:108-129 step, against the gradient digests of
    the unmodified reference (tests/golden/train_step_grads.npz)."""
    import os
    from melgan_multi_b200 import models
    gg = np.load(os.path.join(os.path.dirname(__file__), "golden", "train_step_grads.npz"))
    c = train_case()
    gen = models.Generator()
    gen.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    msd = models.MultiScaleDiscriminator()
    msd.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
    x = torch.from_numpy(synth.mel_input(c["B"], c["T"], c["mel_seed"]))
    y = torch.from_numpy(synth.audio_input(c["B"], 256 * c["T"], c["audio_seed"]))

    def leaves(m):
        vs, gs_, bs = m._param_triplets()
        return [t for trip in zip(vs, gs_, bs) for t in trip]

    def disc(y_, y_hat):
        B = y_.shape[0]
        outs = msd._torch_forward(torch.cat([y_, y_hat]), leaves(msd))
        fm = [outs[7 * s:7 * s + 7] for s in range(3)]
        return ([sc[6][:B].flatten(1) for sc in fm], [sc[6][B:].flatten(1) for sc in fm],
                [[f[:B] for f in sc] for sc in fm], [[f[B:] for f in sc] for sc in fm])

    y_ghat = gen._torch_forward(x, leaves(gen))
    dr, dg, fr, fg = disc(y, y_ghat)
    loss_gen = ref_generator_loss(dg) + ref_feature_loss(fr, fg)
    loss_gen.backward()
    assert abs(loss_gen.item() / float(gg["loss_gen"]) - 1) < 1e-5
    check_grad_digest(gg, "gstep/G/", gen.named_parameters(), 2e-4)
    check_grad_digest(gg, "gstep/D/", msd.named_parameters(), 2e-4)
    msd.zero_grad()
    dr, dg, _, _ = disc(y, y_ghat.detach())
    loss_disc, _, _ = ref_discriminator_loss(dr, dg)
    loss_disc.backward()
    assert abs(loss_disc.item() / float(gg["loss_disc"]) - 1) < 1e-5
    check_grad_digest(gg, "dstep/D/", msd.named_parameters(), 2e-4)


def test_mel_tables_match_the_oracle_filterbank():
    """mg_mel_tables_build (host code of the library: window, twiddles, sparse Slaney filter bank) against oracle/mel_oracle.py."""
    from oracle import mel_oracle as mo
    L = engine.lib()
    L.mg_mel_tables_bytes.restype = ctypes.c_size_t
    n = L.mg_mel_tables_bytes()
    for norm, onorm in ((1, 1), (0, None), (2, "l1")):
        buf = np.zeros((n + 3) // 4, np.float32)
        assert L.mg_mel_tables_build(22050, 80, ctypes.c_float(55), ctypes.c_float(9000), norm, buf.ctypes.data_as(ctypes.c_void_p)) == 0
        ib = buf.view(np.int32)
        win, tw = buf[:1024], buf[1024:2048].reshape(512, 2)
        k = np.arange(1024)
        assert np.abs(win - (0.5 - 0.5 * np.cos(2 * np.pi * k / 1024))).max() < 1e-7
        assert np.abs(tw[:, 0] - np.cos(2 * np.pi * k[:512] / 1024)).max() < 1e-7 and np.abs(tw[:, 1] + np.sin(2 * np.pi * k[:512] / 1024)).max() < 1e-7
        assert ib[2048] == 80
        ks, kc, wo = ib[2049:2049 + 128], ib[2049 + 128:2049 + 256], ib[2049 + 256:2049 + 384]
        wts = buf[2049 + 384:2049 + 384 + 1026]
        dense = np.zeros((80, 513), np.float32)
        for m in range(80):
            dense[m, ks[m]:ks[m] + kc[m]] = wts[wo[m]:wo[m] + kc[m]]
        ref = mo.mel_filterbank(22050, 1024, 80, 55, 9000, norm=onorm)
        assert np.abs(dense - ref).max() <= 2e-7 * max(ref.max(), 1e-30) + 1e-9, (norm, np.abs(dense - ref).max())
    assert L.mg_mel_tables_build(22050, 200, ctypes.c_float(55), ctypes.c_float(9000), 1, buf.ctypes.data_as(ctypes.c_void_p)) == -1
    # every setting of the GPU option sweep (tests/test_mel_isolation_gpu.py) against the float64 filter bank: the sparse
    # runs hold exactly the positive bins, and each weight is its float64 value to fp32 rounding
    for sr, n_mels, fmin, fmax, norm in mel_option_cases():
        assert L.mg_mel_tables_build(sr, n_mels, ctypes.c_float(fmin), ctypes.c_float(fmax), norm, buf.ctypes.data_as(ctypes.c_void_p)) == 0
        ib = buf.view(np.int32)
        assert ib[2048] == n_mels
        ks, kc, wo = ib[2049:2049 + 128], ib[2049 + 128:2049 + 256], ib[2049 + 256:2049 + 384]
        wts = buf[2049 + 384:2049 + 384 + 1026]
        ref = mo.mel_filterbank64(sr, 1024, n_mels, fmin, fmax, NORMS[norm])
        dense = np.zeros((n_mels, 513))
        for m in range(n_mels):
            assert (kc[m] == 0) == (ref[m].max() == 0), (sr, n_mels, norm, m)   # filters that cover no bin
            dense[m, ks[m]:ks[m] + kc[m]] = wts[wo[m]:wo[m] + kc[m]]
        # 2 ulps of each weight (L1: rounded once to float, divided, rounded again); a bin whose float64 weight is a
        # rounding residue (the last filter's top bin at fmax = sr/2) may differ by that residue
        tol = 2 * 2.0 ** -24 * ref + 1e-12 * ref.max(axis=1, keepdims=True)
        assert (np.abs(dense - ref) <= tol).all(), (sr, n_mels, fmin, fmax, norm, float((np.abs(dense - ref) / tol).max()))
    assert L.mg_mel_frames(8192) == 32 and L.mg_mel_frames(255) == 0 and L.mg_mel_frames(256) == 1 and L.mg_mel_frames(1000) == 3
    from melgan_multi_b200 import meldataset
    with pytest.raises(engine.EngineError):
        meldataset.mel_spectrogram(torch.zeros(8192), 1024, 80, 22050, 256, 1024, 55, 9000)


def test_no_test_module_imports_another():
    """Test modules share code through kernel_model (or conftest), never by importing each other: a test file can then be
    renamed or split without breaking unrelated ones."""
    bad = []
    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "test_*.py"))):
        for node in ast.walk(ast.parse(open(path).read(), path)):
            if isinstance(node, ast.Import):
                names = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom) and not node.level:
                names = [node.module]
            else:
                continue
            bad += ["%s:%d imports %s" % (os.path.basename(path), node.lineno, n) for n in names if n.startswith("test_")]
    assert not bad, bad


class _Pinned(torch.Tensor):
    def pin_memory(self):
        return self


def stand_in_cuda():
    """(cuda, torch) stand-ins for what engine._PerStream and engine._StatusWatch call: the current stream's handle is
    cuda.stream; an event has completed when its `done` is set (cuda.done_default for new ones)."""
    import types

    class Event:
        def __init__(self):
            self.done = cuda.done_default

        def record(self, stream=None):
            self.done = cuda.done_default

        def query(self):
            return self.done

        def synchronize(self):
            assert self.done

    class Cuda:
        stream, capturing, done_default, Event = 0, False, True, None

        def current_stream(self, device=None):
            return types.SimpleNamespace(cuda_stream=self.stream)

        def is_current_stream_capturing(self):
            return self.capturing

    cuda = Cuda()
    cuda.Event = Event
    fake = types.SimpleNamespace(cuda=cuda, int32=torch.int32, float32=torch.float32,
                                 zeros=lambda n, dtype, device=None: torch.zeros(n, dtype=dtype).as_subclass(_Pinned),
                                 empty=lambda n, dtype, device=None: torch.empty(n, dtype=dtype))
    return cuda, fake


def test_per_stream_scratch_is_private_bounded_and_keeps_graph_buffers():
    """engine._PerStream on a stand-in for torch.cuda: each stream has its own scratch, a stream's buffer grows in place
    of the old one, the least recently used stream beyond LIMIT is dropped, and a buffer used while a CUDA graph was being
    captured stays allocated after its stream is dropped."""
    cuda, fake = stand_in_cuda()
    per = engine._PerStream(fake, "cuda:0", "test")
    bufs = {}
    for s in range(1, per.LIMIT + 1):
        cuda.stream = s
        cuda.capturing = s == 2
        bufs[s] = per.current().buffer("ws", 64)
    cuda.capturing = False
    assert len({id(b) for b in bufs.values()}) == per.LIMIT
    cuda.stream = 1
    assert per.current().buffer("ws", 64) is bufs[1] and per.current().buffer("ws", 16) is bufs[1]
    grown = per.current().buffer("ws", 65)
    assert grown is not bufs[1] and grown.numel() * 4 >= 65 and per.current().bufs["ws"] is grown
    cuda.stream = per.LIMIT + 1  # stream 2 is now the least recently used: dropped, its captured buffer held
    per.current().buffer("ws", 64)
    assert 2 not in per._by_stream and 1 in per._by_stream and len(per._by_stream) == per.LIMIT
    assert len(per._held) == 1 and per._held[0] is bufs[2]
    status = per.current().buffer("status", 256, zeros=True)
    assert status.dtype == torch.int32 and status.numel() == 64 and not status.any()


def test_status_watches_of_dropped_streams_are_bounded_and_reported():
    """A server that takes a new stream per request rotates through more streams than _PerStream.LIMIT.  The watches of
    dropped streams must be checked at the module's next call and reused once their copy has landed: the pinned slots
    and events stay bounded, and a timed-out wait of a call whose stream was dropped raises at the next call."""
    cuda, fake = stand_in_cuda()
    per = engine._PerStream(fake, "cuda:0", "test")

    def call(stream, code=0):  # one forward's status handling, as GeneratorDevice.forward does it
        cuda.stream = stream
        sc = per.current()
        sc.check()
        word = sc.buffer("status", 4, zeros=True)
        word.fill_(code)
        sc.arm(word[:1])
        return sc.watch

    n_streams = per.LIMIT + 9
    watches = {id(call(1 + k % n_streams)) for k in range(10 * n_streams)}
    assert len(per._by_stream) == per.LIMIT
    assert len(watches) <= per.LIMIT + 1, len(watches)
    assert len(per._retired) <= per.LIMIT + 1
    # a timed-out wait on stream 1000 whose copy is still in flight when 1000 is dropped
    cuda.done_default = False
    slow = call(1000, code=7)
    cuda.done_default = True
    for k in range(per.LIMIT):
        call(2000 + k)
    assert 1000 not in per._by_stream and any(w is slow for w in per._retired)
    slow.event.done = True  # the copy lands
    with pytest.raises(engine.EngineError, match="role code 7"):
        call(3000)
    call(3001)  # reported once
    assert not slow.pending and len(per._retired) <= per.LIMIT + 1
