"""The memory-bound building blocks of the vision and text towers, per element against fp64 (tests/tower_blocks_oracle.py
derives every bound), at the sizes production batches run at.

Each of these kernels is a grid-stride loop whose grid is capped by the SM count, so a warp (or thread) only handles more
than one row past that cap: 16 blocks x 8 warps per SM for the forward LayerNorms, 8 x 8 for the LayerNorm backward.  The
row counts below are derived from pg_device_sm_count() so that both sides of every cap are run.  Outputs are surrounded by
NaN guard rows or columns that must survive every call.

Forward kernels without an entry point of their own (im2col, embed_preln, token_mean, text_embed, the pooling LayerNorm) are
checked through pg_vit_forward_train / pg_text_forward_train, whose saved activations are read back from the arena."""
import ctypes as C

import pytest
import torch

import tower_blocks_oracle as O

pytestmark = pytest.mark.gpu

EPS = 1e-5
HIDDENS = [128, 256, 512, 768, 1024]
SENT = {torch.float32: (0x7FD5A5A5, torch.int32), torch.float16: (0x7E5A, torch.int16), torch.bfloat16: (0x7FD5, torch.int16)}
RATIOS = {}


@pytest.fixture(scope="module")
def env(cuda):
    from pigeon_b200 import _lib
    lib = _lib.load()
    sms = int(lib.pg_device_sm_count())
    assert sms > 0
    yield lib, sms, _lib.check, _lib.ptr, _lib.current_stream_ptr
    if RATIOS:
        print("\nlargest |error| / bound per kernel:", {k: f"{v:.3g}" for k, v in sorted(RATIOS.items())})


def _note(key, err, bound):
    r = O.ratio(err, bound)
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    assert r <= 1.0, (key, r)


class Guarded:
    """A [rows, cols] tensor inside a buffer of sentinel NaNs: `guard` rows above and below and `pad` columns on the right."""

    def __init__(self, rows, cols, dtype, device, guard=1, pad=0, fill=None):
        self.rows, self.cols, self.guard, self.ld = rows, cols, guard, cols + pad
        bits, idt = SENT[dtype]
        self.buf = torch.full(((rows + 2 * guard) * self.ld,), bits, dtype=idt, device=device).view(dtype)
        self.t = self.buf[guard * self.ld:(guard + rows) * self.ld].view(rows, self.ld)[:, :cols]
        if isinstance(fill, float):
            self.t.fill_(fill)
        elif fill is not None:
            self.t.copy_(fill)

    def ptr(self):
        return self.t.data_ptr()

    def intact(self):
        bits, idt = SENT[self.buf.dtype]
        full = self.buf.view(idt).view(-1, self.ld)
        g = self.guard
        ok = bool((full[:g] == bits).all()) and bool((full[g + self.rows:] == bits).all())
        return ok and bool((full[g:g + self.rows, self.cols:] == bits).all())


def _ln_input(rows, hidden, device, gen):
    """Rows cycle through four kinds: plain, a large common offset (1000 + N(0, 1)), constant, one outlier channel at 150."""
    x = torch.randn(rows, hidden, device=device, generator=gen) * 2 + 0.3
    kind = torch.arange(rows, device=device) % 4
    x[kind == 1] = 1000 + torch.randn(int((kind == 1).sum()), hidden, device=device, generator=gen)
    x[kind == 2] = (0.7 + 0.01 * (torch.arange(rows, device=device)[kind == 2] % 97).float())[:, None]
    x[kind == 3, 7] = 150.0
    g = 1 + 0.2 * torch.randn(hidden, device=device, generator=gen)
    b = 0.1 * torch.randn(hidden, device=device, generator=gen)
    return x, g, b


def _fwd_rows(sms, f16):
    cap = 16 * 8 * sms
    out = [1, 7, 577, cap, cap + 1]
    return out + [256 * 577] if f16 else out


# ------------------------------------------------------------------------------------------------ LayerNorm forward
@pytest.mark.parametrize("hidden", HIDDENS)
@pytest.mark.parametrize("f16", [True, False])
def test_layernorm_forward_per_element(env, cuda, hidden, f16):
    lib, sms, check, ptr, sp = env
    gen = torch.Generator(device=cuda).manual_seed(hidden + f16)
    for rows in _fwd_rows(sms, f16):
        x, g, b = _ln_input(rows, hidden, cuda, gen)
        y = Guarded(rows, hidden, torch.float16 if f16 else torch.float32, cuda)
        fn = lib.pg_layernorm_f16 if f16 else lib.pg_layernorm_f32
        check(fn(ptr(x), y.ptr(), ptr(g), ptr(b), rows, hidden, EPS, sp()), "layernorm")
        ref, bound = O.layernorm_forward(x, g, b, EPS, out_f16=f16)
        assert y.intact(), rows
        _note("layernorm_f16" if f16 else "layernorm_f32", y.t.double() - ref, bound)


@pytest.mark.parametrize("hidden", [384, 640, 2048, 100])
def test_layernorm_forward_refuses_unsupported_hidden(env, cuda, hidden):
    lib, sms, check, ptr, sp = env
    x = torch.randn(5, hidden, device=cuda)
    g, b = torch.ones(hidden, device=cuda), torch.zeros(hidden, device=cuda)
    for dt, fn in ((torch.float16, lib.pg_layernorm_f16), (torch.float32, lib.pg_layernorm_f32)):
        y = Guarded(5, hidden, dt, cuda, guard=0)
        assert fn(ptr(x), y.ptr(), ptr(g), ptr(b), 5, hidden, EPS, sp()) != 0
        torch.cuda.synchronize()
        assert y.intact(), "nothing may be written"


# ------------------------------------------------------------------------------------------------ LayerNorm backward
@pytest.mark.parametrize("hidden", HIDDENS)
def test_layernorm_backward_per_element(env, cuda, hidden):
    lib, sms, check, ptr, sp = env
    cap = 8 * 8 * sms
    gen = torch.Generator(device=cuda).manual_seed(hidden)
    for rows in (5, 1000, cap, cap + 1, 64 * 577):
        x, gamma, _ = _ln_input(rows, hidden, cuda, gen)
        dy = torch.randn(rows, hidden, device=cuda, generator=gen) * 1e-3
        dx0 = torch.randn(rows, hidden, device=cuda, generator=gen) * 1e-3
        dg0 = torch.randn(hidden, device=cuda, generator=gen) * 0.5
        db0 = torch.randn(hidden, device=cuda, generator=gen) * 0.5
        blocks, rpw = O.ln_backward_schedule(rows, sms)
        for accumulate in (1, 0):
            ref = O.layernorm_backward(dy, x, gamma, EPS, dx0=dx0 if accumulate else None)
            for params in (True, False):
                dx = Guarded(rows, hidden, torch.float32, cuda, fill=dx0 if accumulate else float("nan"))
                d16 = Guarded(rows, hidden, torch.bfloat16, cuda)
                dg = Guarded(1, hidden, torch.float32, cuda, fill=dg0[None])
                db = Guarded(1, hidden, torch.float32, cuda, fill=db0[None])
                check(lib.pg_layernorm_backward(ptr(dy), ptr(x), ptr(gamma), dx.ptr(), accumulate,
                                                dg.ptr() if params else None, db.ptr() if params else None,
                                                d16.ptr() if accumulate else None, rows, hidden, EPS, sp()),
                      "pg_layernorm_backward")
                assert dx.intact() and d16.intact() and dg.intact() and db.intact(), (rows, accumulate, params)
                _note("layernorm_backward dx", dx.t.double() - ref["dx"], ref["bound"])
                if accumulate:
                    assert torch.equal(d16.t, dx.t.to(torch.bfloat16)), "dx_bf16 must be bf16(dx)"
                if params:
                    bg, bb = O.ln_param_bounds(ref, dg0, db0, rpw + 8 + blocks)
                    _note("layernorm_backward dgamma", dg.t[0].double() - (dg0.double() + ref["dgamma"]), bg)
                    _note("layernorm_backward dbeta", db.t[0].double() - (db0.double() + ref["dbeta"]), bb)
                else:
                    assert torch.equal(dg.t[0], dg0) and torch.equal(db.t[0], db0)


# ------------------------------------------------------------------------------------------------ column sums
@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("rows", [1, 127, 128, 129, 36928])
def test_column_sum_accumulate(env, cuda, rows, bf16):
    lib, sms, check, ptr, sp = env
    gen = torch.Generator(device=cuda).manual_seed(rows)
    dt = torch.bfloat16 if bf16 else torch.float32
    for cols in (1, 255, 256, 257, 3072, 4096):
        ldx = cols + 3
        x = (torch.randn(rows, ldx, device=cuda, generator=gen) + 0.25).to(dt)
        x[:, cols:] = float("nan")                                    # beyond cols: never read
        out0 = torch.randn(cols, device=cuda, generator=gen)
        out = Guarded(1, cols, torch.float32, cuda, pad=4, fill=out0[None])
        check(lib.pg_column_sum_accumulate(ptr(x), 2 if bf16 else 0, ldx, out.ptr(), rows, cols, sp()),
              "pg_column_sum_accumulate")
        ref, bound = O.column_sum(x[:, :cols], out0)
        assert out.intact(), cols
        _note("column_sum_accumulate", out.t[0].double() - ref, bound)


# ------------------------------------------------------------------------------------------------ token mean backward
@pytest.mark.parametrize("tokens", [1, 77, 577])
def test_token_mean_backward_is_exact(env, cuda, tokens):
    lib, sms, check, ptr, sp = env
    gen = torch.Generator(device=cuda).manual_seed(tokens)
    n = 3
    for hidden in (100, 128, 1024):
        d = torch.randn(n, hidden, device=cuda, generator=gen)
        g = Guarded(n * tokens, hidden, torch.float32, cuda)
        check(lib.pg_token_mean_backward(ptr(d), g.ptr(), n, tokens, hidden, sp()), "pg_token_mean_backward")
        inv = torch.tensor(1.0, dtype=torch.float32) / tokens
        ref = (d * inv.to(cuda))[:, None, :].expand(n, tokens, hidden).reshape(n * tokens, hidden)
        assert g.intact() and torch.equal(g.t, ref), hidden
    g = Guarded(n * tokens, 102, torch.float32, cuda)
    assert lib.pg_token_mean_backward(ptr(torch.zeros(n, 102, device=cuda)), g.ptr(), n, tokens, 102, sp()) != 0
    torch.cuda.synchronize()
    assert g.intact()


# ------------------------------------------------------------------------------------------------ embedding backward
@pytest.mark.parametrize("n_views", [1, 3, 64])
def test_embed_backward_is_the_ascending_view_sum(env, cuda, n_views):
    lib, sms, check, ptr, sp = env
    gen = torch.Generator(device=cuda).manual_seed(n_views)
    for tokens in (5, 77, 257, 577):
        for hidden in HIDDENS:
            de = torch.randn(n_views, tokens, hidden, device=cuda, generator=gen)
            pos0 = torch.randn(tokens, hidden, device=cuda, generator=gen)
            cls0 = torch.randn(hidden, device=cuda, generator=gen)
            s = torch.zeros(tokens, hidden, device=cuda)
            for v in range(n_views):
                s = s + de[v]
            dpos = Guarded(tokens, hidden, torch.float32, cuda, fill=pos0)
            dcls = Guarded(1, hidden, torch.float32, cuda, fill=cls0[None])
            check(lib.pg_embed_backward(ptr(de), dpos.ptr(), dcls.ptr(), n_views, tokens, hidden, sp()), "pg_embed_backward")
            assert dpos.intact() and dcls.intact()
            assert torch.equal(dpos.t, pos0 + s) and torch.equal(dcls.t[0], cls0 + s[0]), (tokens, hidden)
            dpos2 = Guarded(tokens, hidden, torch.float32, cuda, fill=pos0)
            sentinel = Guarded(1, hidden, torch.float32, cuda, fill=cls0[None])
            check(lib.pg_embed_backward(ptr(de), dpos2.ptr(), None, n_views, tokens, hidden, sp()), "pg_embed_backward")
            assert torch.equal(dpos2.t, pos0 + s) and dpos2.intact()
            assert torch.equal(sentinel.t[0], cls0) and sentinel.intact()


# ------------------------------------------------------------------------------------------------ text pooling LN backward
def _pool_ids(n, S, device, gen, vocab=49408):
    """Caption b puts its largest id at t = 0 (b % 3 == 0), at t = S - 1 (b % 3 == 1) or at two tied positions (b % 3 == 2)."""
    ids = torch.randint(1, vocab - 1, (n, S), device=device, generator=gen)
    for b in range(n):
        if b % 3 == 0:
            ids[b, 0] = vocab - 1
        elif b % 3 == 1:
            ids[b, S - 1] = vocab - 1
        else:
            t = (b * 7) % S
            ids[b, t] = vocab - 1
            ids[b, min(S - 1, t + 1 + b % 5)] = vocab - 1
    return ids


@pytest.mark.parametrize("hidden", [512, 768, 1024])
@pytest.mark.parametrize("n", [1, 7, 9, 256])
def test_text_pool_ln_backward(env, cuda, n, hidden):
    lib, sms, check, ptr, sp = env
    gen = torch.Generator(device=cuda).manual_seed(n * hidden)
    for S in (1, 2, 77):
        ids = _pool_ids(n, S, cuda, gen)
        x, gamma, _ = _ln_input(n * S, hidden, cuda, gen)
        dp = torch.randn(n, hidden, device=cuda, generator=gen) * 1e-2
        dg0 = torch.randn(hidden, device=cuda, generator=gen)
        db0 = torch.randn(hidden, device=cuda, generator=gen)
        runs = []
        for _ in range(2):
            g = Guarded(n * S, hidden, torch.float32, cuda)
            part = torch.empty(n, 2 * hidden, device=cuda)
            dg = Guarded(1, hidden, torch.float32, cuda, fill=dg0[None])
            db = Guarded(1, hidden, torch.float32, cuda, fill=db0[None])
            check(lib.pg_text_pool_ln_backward(ptr(x), ptr(dp), ptr(gamma), ptr(ids), n, S, hidden, EPS, g.ptr(), ptr(part),
                                               dg.ptr(), db.ptr(), sp()), "pg_text_pool_ln_backward")
            assert g.intact() and dg.intact() and db.intact()
            runs.append((g.t.clone(), dg.t.clone(), db.t.clone()))
        assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(*runs)), "two runs, same bits"
        g_out, dg_out, db_out = runs[0]
        rows = torch.arange(n, device=cuda) * S + O.first_argmax(ids)
        ref = O.layernorm_backward(dp, x[rows], gamma, EPS)
        _note("text_pool_ln_backward dx", g_out[rows].double() - ref["dx"], ref["bound"])
        others = torch.ones(n * S, dtype=torch.bool, device=cuda)
        others[rows] = False
        assert torch.equal(g_out[others].view(torch.int32), torch.full_like(g_out[others].view(torch.int32),
                                                                            SENT[torch.float32][0])), "other rows untouched"
        bg, bb = O.ln_param_bounds(ref, dg0, db0, n + 1)
        _note("text_pool_ln_backward dgamma", dg_out[0].double() - (dg0.double() + ref["dgamma"]), bg)
        _note("text_pool_ln_backward dbeta", db_out[0].double() - (db0.double() + ref["dbeta"]), bb)


# ------------------------------------------------------------------------------------------------ token embedding gradient
def test_token_embedding_grad(env, cuda):
    lib, sms, check, ptr, sp = env
    n, S, hidden, vocab, pad = 256, 77, 512, 49408, 0
    gen = torch.Generator(device=cuda).manual_seed(5)
    ids = torch.randint(1, vocab - 1, (n, S), device=cuda, generator=gen)
    lengths = torch.randint(2, S, (n,), device=cuda, generator=gen)
    t = torch.arange(S, device=cuda)[None]
    ids = torch.where(t == lengths[:, None], vocab - 1, ids)             # one EOT (vocab - 1) per caption
    ids = torch.where(t > lengths[:, None], pad, ids)                    # padding: thousands of rows of one id
    ids[3, 5], ids[40, 0], ids[77, 60] = -1, vocab, vocab                # outside the vocabulary
    ids = ids.reshape(-1).contiguous()
    assert int((ids == pad).sum()) > 2000
    dx = torch.randn(n * S, hidden, device=cuda, generator=gen)
    dx[(ids < 0) | (ids >= vocab)] = float("nan")
    dtok0 = torch.randn(vocab, hidden, device=cuda, generator=gen)
    ref, bound, seen = O.token_embedding_grad(ids, dx, vocab, dtok0)
    runs = []
    for _ in range(2):
        dtok = Guarded(vocab, hidden, torch.float32, cuda, fill=dtok0)
        check(lib.pg_token_embedding_grad(ptr(ids), ptr(dx), n * S, hidden, vocab, dtok.ptr(), sp()), "pg_token_embedding_grad")
        assert dtok.intact()
        runs.append(dtok.t.clone())
    assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32)), "two runs, same bits"
    out = runs[0]
    assert torch.isfinite(out).all()
    assert torch.equal(out[~seen].view(torch.int32), dtok0[~seen].view(torch.int32)), "ids that never occur are unchanged"
    _note("token_embedding_grad", out[seen].double() - ref[seen], bound[seen])


# ------------------------------------------------------------------------------------------------ vision forward
def _arena(tr, addr, shape, dtype):
    nbytes = int(torch.Size(shape).numel()) * torch.empty((), dtype=dtype).element_size()
    off = addr - tr._arena.data_ptr()
    return tr._arena[off:off + nbytes].view(dtype).view(shape)


@pytest.mark.parametrize("hidden,image,patch,px16", [(h, 336, 14, False) for h in HIDDENS[1:]] +   # pg_vit_create: hidden % 256
                         [(256, 224, 16, False), (512, 336, 14, True)])
def test_vision_forward_blocks(env, cuda, hidden, image, patch, px16):
    lib, sms, check, ptr, sp = env
    from pigeon_b200 import CLIPVisionTower, VitDims, synthetic
    from pigeon_b200.vit_train import TowerTrainer
    dims = VitDims(image_size=image, patch_size=patch, hidden=hidden, heads=hidden // 64, intermediate=4 * hidden, layers=1)
    T, np_, K, Kp = dims.tokens, dims.tokens - 1, dims.patch_k, dims.patch_k_pad
    n = max(30, (16 * 8 * sms) // T + 1)                                   # past the LayerNorm grid cap
    assert n * T > 16 * 8 * sms and n * np_ * Kp // 8 > 16 * sms * 256     # and past im2col's
    sd = synthetic.random_vit_state_dict(dims, seed=hidden + image, std=0.05)
    tower = CLIPVisionTower(dims)
    tower.load_state_dict(sd, strict=True)
    tower.to(cuda)
    tr = TowerTrainer(tower, max_views=n)
    gen = torch.Generator(device=cuda).manual_seed(hidden)
    px = torch.randn(n, 3, image, image, device=cuda, generator=gen) * 1.5
    px = px.half() if px16 else px
    tr._build_saved(n)
    emb = Guarded(n, hidden, torch.float32, cuda)
    check(lib.pg_vit_forward_train(tower.engine()._handle, ptr(px), int(px16), n, C.byref(tr._saved), emb.ptr(), sp()),
          "pg_vit_forward_train")
    torch.cuda.synchronize()
    assert emb.intact()
    p = {k.replace("vision_model.", ""): v.to(cuda) for k, v in sd.items()}

    a16 = _arena(tr, tr._saved.im2col, (n * np_, Kp), torch.float16)
    cols = torch.nn.functional.unfold(px.half().float(), patch, stride=patch).transpose(1, 2).reshape(n * np_, K).half()
    assert torch.equal(a16[:, :K].view(torch.int16), cols.view(torch.int16)), "im2col"
    assert (a16[:, K:].view(torch.int16) == 0).all(), "im2col padding columns are +0"

    e = _arena(tr, tr._saved.e, (n, T, hidden), torch.float32)
    cls, pos = p["embeddings.class_embedding"], p["embeddings.position_embedding.weight"]
    assert torch.equal(e[:, 0], (cls + pos[0]).expand(n, hidden)), "class token"
    w16 = p["embeddings.patch_embedding.weight"].reshape(hidden, K).half()
    ref, bound = O.patch_embedding(a16[:, :K], w16, pos[1:].repeat(n, 1))
    _note("patch embedding (GEMM + embed_preln)", e[:, 1:].reshape(-1, hidden).double() - ref, bound)

    L = tr._saved_layers[0]
    x0 = _arena(tr, L.x0, (n * T, hidden), torch.float32)
    ref, bound = O.layernorm_forward(e.reshape(-1, hidden), p["pre_layrnorm.weight"], p["pre_layrnorm.bias"], EPS)
    _note("embed_preln", x0.double() - ref, bound)
    xn1 = _arena(tr, L.xn1, (n * T, hidden), torch.float16)
    ref, bound = O.layernorm_forward(x0, p["encoder.layers.0.layer_norm1.weight"], p["encoder.layers.0.layer_norm1.bias"], EPS,
                                     out_f16=True)
    _note("layernorm_f16 (layer 0 xn1)", xn1.double() - ref, bound)
    x_out = _arena(tr, tr._saved.x_out, (n, T, hidden), torch.float32)
    ref, bound = O.token_mean(x_out, hidden)
    _note("token_mean", emb.t.double() - ref, bound)


# ------------------------------------------------------------------------------------------------ text forward
@pytest.mark.parametrize("hidden", [512, 768])
def test_text_forward_blocks(env, cuda, hidden):
    lib, sms, check, ptr, sp = env
    from pigeon_b200.clip_text import CLIPTextTower, TextDims
    from pigeon_b200.clip_train import TextTrainer
    n, S, vocab = 256, 77, 49408
    dims = TextDims(vocab=vocab, max_positions=S, hidden=hidden, heads=hidden // 64, intermediate=4 * hidden, layers=1)
    tower = CLIPTextTower(dims).to(cuda)
    gen = torch.Generator(device=cuda).manual_seed(hidden)
    with torch.no_grad():
        for name, q in tower.named_parameters():
            q.copy_(torch.randn(q.shape, device=cuda, generator=gen) * 0.05 + (1.0 if "norm" in name and "weight" in name else 0.0))
    tr = TextTrainer(tower)
    ids = _pool_ids(n, S, cuda, gen, vocab)
    tm = tower.text_model
    tok, pos = tm.embeddings.token_embedding.weight.detach(), tm.embeddings.position_embedding.weight.detach()

    def run(ids):
        tr._build_saved(n, S)
        pooled = Guarded(n, hidden, torch.float32, cuda)
        check(lib.pg_text_forward_train(tower.engine()._handle, ptr(ids), None, n, S, C.byref(tr._saved), pooled.ptr(), sp()),
              "pg_text_forward_train")
        torch.cuda.synchronize()
        assert pooled.intact()
        return pooled, _arena(tr, tr._saved_layers[0].x0, (n * S, hidden), torch.float32)

    pooled, x0 = run(ids)
    assert n * S > 16 * 8 * sms
    assert torch.equal(x0, (tok[ids] + pos[:S][None]).reshape(n * S, hidden)), "x0 = tok[id] + pos[t]"
    x_final = _arena(tr, tr._saved.x_final, (n, S, hidden), torch.float32)
    rows = x_final[torch.arange(n, device=cuda), O.first_argmax(ids)]
    ref, bound = O.layernorm_forward(rows, tm.final_layer_norm.weight.detach(), tm.final_layer_norm.bias.detach(), EPS)
    _note("text pooled LayerNorm", pooled.t.double() - ref, bound)

    bad = ids.clone()
    bad[5, 3] = vocab
    _, x0 = run(bad)
    finite = torch.isfinite(x0).all(1)
    assert torch.isnan(x0[5 * S + 3]).all() and int((~finite).sum()) == 1
