"""Every stage of the refiner and scorer heads in place, at the batch sizes the product runs, against float64 references
on the GPU.

fp_op_heads runs the product's own run_refine_heads / run_score_feats on given tokens and returns one stage's whole
workspace buffer, so each stage is checked on the buffers, group offsets, streams and tiles the product uses.  Each
stage's float64 reference (tests/heads_reference.py) is computed from the GPU's own previous stage, so errors do not
compound, with the weights exactly as engine.pack_network uploads them:
  refiner  qkv = tok Win^T + b;  att of each group on the GPU's qkv columns 1536 g + (0, 512, 1024);
           x1pre = att_g Wout^T + b + tok;  x1 = LayerNorm1(x1pre);  ff = relu(x1 W1^T + b1);  x2pre = ff W2^T + b2 + x1;
           head_out = fin . mean_t LayerNorm2(x2pre) + b
  scorer   qkv;  att (one group);  tok_mean = mean_t att;  feats = out_proj(tok_mean)
The tokens are drawn once, by the encoder at N = 512 on random crops, and sliced: every N sees identical inputs.

Grid: the refiner at N = 1 (track_one: the 128 x 128 tile, heads forked onto two streams), 32 (a shard: the
in-projection on linear_ws_kernel, the 512-wide layers on the 128 tile), 67 (M mod 64 = 48, forked), 249 (the last
64-row tile holds 16 rows), 252 and 512 (kRegisterPassCap); the scorer at 1, 32, 249 and 512.  Only the 3072-wide
in-projection has CTAs whose range crosses a weight-panel boundary (12 per launch on 132 SMs).
"""
import time

import pytest
import torch
import torch.nn.functional as F

import heads_reference as ref

pytestmark = pytest.mark.gpu

N_MAX = 512
REFINE_N = (1, 32, 67, 249, 252, 512)
SCORE_N = (1, 32, 249, 512)
REFINE_STAGES = ("qkv", "att", "x1pre", "x1", "ff", "x2pre", "head_out")
SCORE_STAGES = ("qkv", "att", "tok_mean", "feats")
CHUNK = 16  # hypotheses per block of the float64 references

PROBES = {
    "a": "K block 448..511 dropped",
    "b": "residual omitted",
    "b'": "residual taken from x1pre instead of x1",
    "c": "bias of the neighbouring 128-channel panel",
    "d": "group 1 computed from group 0's input",
    "e": "no ReLU",
    "f": "last 64-row tile computed from the previous tile's rows",
    "t": "token mean over 399",
}
# Least fraction of the compared elements each probe must fail on (f: of the last tile's elements; d: of group 1's),
# below the ranges measured on an H100 (see test_refiner_stages).  FF1 sets the floor of (a), (c), (d) and (f): where
# ReLU clamps both the reference and the probe to zero they agree.
PROBE_MIN = {"a": 0.45, "b": 0.9, "b'": 0.9, "c": 0.4, "d": 0.55, "e": 0.35, "f": 0.45, "t": 0.9}


@pytest.fixture(autouse=True)
def _release_cached_memory():
    # the float64 references are large: hand their cached blocks back to the device after each test
    yield
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def setup():
    from foundationpose_b200.engine import Engine, crops_from_planar, pack_network
    from foundationpose_b200.weights import random_state_dict

    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    e = Engine()
    gen = torch.Generator(device="cuda").manual_seed(4096)
    A = torch.rand(N_MAX, 6, 160, 160, generator=gen, device="cuda")
    B = torch.rand(N_MAX, 6, 160, 160, generator=gen, device="cuda")
    for T in (A, B):
        T[:, 3:] = (T[:, 3:] - 0.5) * 2
        T[:, 3:, :30] = 0
    crops = crops_from_planar(A, B)
    del A, B
    weights, tokens = {}, {}
    for kind, seed in (("refine", 7), ("score", 8)):
        sd = random_state_dict(kind, seed)
        e.load_network(kind, sd)
        weights[kind] = {k: torch.from_numpy(v).cuda() for k, v in pack_network(sd, kind).items()}
        tokens[kind] = e.op_tokens(kind, crops, N_MAX)
    del crops
    yield e, weights, tokens
    print(f"\nheads stage tests: {time.time() - t0:.1f} s, peak torch allocation "
          f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB ({torch.cuda.get_device_name()})")
    e.close()


class _Stage:
    """Worst error / bar of one stage, where it first went over the bar, and its probes' failure counts."""

    def __init__(self, name):
        self.name, self.ratio, self.over = name, 0.0, None
        self.fails, self.counts = {}, {}

    def check(self, got, y, bar, where):
        got = got.double()
        err = (got - y).abs()
        self.ratio = max(self.ratio, (err / bar).max().item())
        bad = err > bar
        if self.over is None and bad.any():
            idx = tuple(bad.nonzero()[0].tolist())
            self.over = (f"{int(bad.sum())} elements over the bar in {where}, first at {idx}: got {got[idx].item():.6g} "
                         f"ref {y[idx].item():.6g} bar {bar[idx].item():.3g}")

    def probe(self, p, got, wrong, bar):
        self.fails[p] = self.fails.get(p, 0) + int(((got.double() - wrong).abs() > bar).sum())
        self.counts[p] = self.counts.get(p, 0) + got.numel()

    def report(self, what):
        """Prints the stage's line; returns its failures."""
        fr = {p: self.fails[p] / self.counts[p] for p in self.fails}
        probes = ", ".join(f"({p}) {fr[p]:.1%}" for p in sorted(fr))
        print(f"{what} {self.name:8s}: worst error / bar {self.ratio:.3f}" + (f"; probes fail {probes}" if probes else ""))
        bad = [f"{what} {self.name}: {self.over}"] if self.over else []
        bad += [f"{what} {self.name}: probe ({p}) {PROBES[p]} fails only {fr[p]:.2%} (needs > {PROBE_MIN[p]:.0%})"
                for p in fr if fr[p] <= PROBE_MIN[p]]
        return bad


def _linear(stage, got, x, w, b, where, res=None, relu=False, res_alt=None, d=None):
    """One linear stage on a block of rows: got vs relu(x w^T + b + res), and its probes.  d = (x, res) of group 0."""
    acc, mag = ref.linear_terms(x, w)
    y = ref.enc.epilogue(acc, b, res, relu=relu)
    bar = ref.enc.bar(y, acc, mag, b, ref.LINEAR_STEPS, res)
    stage.check(got, y, bar, where)
    drop, _ = ref.linear_terms(x, w, 448, 512)
    stage.probe("a", got, ref.enc.epilogue(acc - drop, b, res, relu=relu), bar)
    stage.probe("c", got, ref.enc.epilogue(acc, ref.neighbour_panel(b), res, relu=relu), bar)
    if res is not None:
        stage.probe("b", got, ref.enc.epilogue(acc, b, None, relu=relu), bar)
    if res_alt is not None:
        stage.probe("b'", got, ref.enc.epilogue(acc, b, res_alt, relu=relu), bar)
    if relu:
        stage.probe("e", got, ref.enc.epilogue(acc, b, res, relu=False), bar)
    if d is not None:
        stage.probe("d", got, ref.enc.epilogue(ref.linear_terms(d[0], w)[0], b, d[1], relu=relu), bar)


def _last_tile(stage, got, x, w, b, M, res=None, relu=False):
    """Probe (f): the rows of the ragged last 64-row tile against a reference that reads the previous tile's rows."""
    r0 = M - M % 64
    acc, mag = ref.linear_terms(x[r0:M], w)
    rs = None if res is None else res[r0:M]
    y = ref.enc.epilogue(acc, b, rs, relu=relu)
    bar = ref.enc.bar(y, acc, mag, b, ref.LINEAR_STEPS, rs)
    stage.probe("f", got[r0:M], ref.enc.epilogue(ref.linear_terms(x[r0 - 64:M - 64], w)[0], b, rs, relu=relu), bar)


def _tiles(M, couts, N):
    """ops.gemm_tile_m of each linear layer: 128 (gemm_tile_kernel) at N = 1, 64 (linear_ws_kernel) at N >= 249."""
    from foundationpose_b200 import _lib, ops

    tiles = {c: ops.gemm_tile_m(_lib.LAYER_LINEAR, n_img=1, Hin=1, Win=M, Cin=512, Cout=c) for c in couts}
    for c, tm in tiles.items():
        if N == 1:
            assert tm == 128, f"N=1: the {c}-wide linear layer takes tile_m {tm}, not the 128 tile"
        if N >= 249:
            assert tm == 64, f"N={N}: the {c}-wide linear layer takes tile_m {tm}, not linear_ws_kernel's 64 rows"
    return ", ".join(f"{c}-wide: tile_m {tm}" for c, tm in tiles.items())


@pytest.mark.parametrize("N", REFINE_N)
def test_refiner_stages(setup, N):
    """Every refiner stage at N hypotheses against its float64 reference on the GPU's previous stage, per element within
    its bar (heads_reference): linear layers encoder_reference.bar with 32 steps, attention 1.25 u16 (|o| + P|V|) + sub,
    LayerNorm its derived bar, head_out TOKEN_BAR_U32 u32 of the L1 magnitude.

    Probes, each a reference wrong in one place, with the least fraction of the compared elements it must fail on
    (PROBE_MIN) and the range measured on an H100 80GB HBM3 (700 W) over the grid of both tests:
      (a) every linear stage: K block 448..511 dropped: 45 % (58.1 % on FF1, 99.6 to 99.8 % on the others);
      (b) out-proj and FF2: residual omitted: 90 % (99.8 to 99.9 %);
      (b') FF2's residual taken from x1pre instead of x1: 90 % (99.9 to 100 %);
      (c) every linear stage: the bias of the neighbouring 128-channel panel: 40 % (51.4 % on FF1, 95.9 to 99.6 % on the
          others and on the scorer's features);
      (d) every per-group stage: group 1's stage computed from group 0's input, of group 1's elements: 55 % (68.6 to
          68.7 % on FF1, 99.9 to 100 % on the others);
      (e) FF1 without ReLU: 35 % (48.2 %);
      (f) N = 1, 67, 249 (M mod 64 = 16, 48, 16): the ragged last 64-row tile of each linear stage computed from the
          previous tile's rows, of the last tile's elements: 45 % (60.1 to 61.2 % on FF1, 98.8 to 99.9 % on the others);
      (t) head_out and the scorer's token mean: the mean over 399 tokens: 90 % (100 %).
    Measured there: at most 0.80 of the bar (LayerNorm 1, where the fp16 rounding of the output dominates), 0.66 to
    0.76 on the linear stages, 0.47 to 0.59 on attention, below 0.03 on the token reductions.
    """
    e, W, TOK = setup
    w = W["refine"]
    t0 = time.time()
    M = N * 400
    tiles = _tiles(M, (3072, 512), N)
    tok = TOK["refine"][:N]
    got = {s: e.op_heads("refine", tok, N, i) for i, s in enumerate(REFINE_STAGES)}
    t = tok.reshape(M, 512)
    st = {s: _Stage(s) for s in REFINE_STAGES}
    H = lambda g, s: w[f"head{g}.{s}"]
    for h0 in range(0, N, CHUNK):
        h1 = min(N, h0 + CHUNK)
        r = slice(h0 * 400, h1 * 400)
        where = f"hypotheses {h0}..{h1 - 1}"
        _linear(st["qkv"], got["qkv"][r], t[r], w["heads.in_w"], w["heads.in_b"], where)
        o0 = None
        for g in range(2):
            wg = f"{where}, group {g}"
            o, pv, sub, _, _ = ref.attention(got["qkv"], N, 2, g, h0, h1)
            bar = ref.attention_bar(o, pv, sub)
            ga = got["att"][g, r].view(h1 - h0, 400, 4, 128)
            st["att"].check(ga, o, bar, wg)
            if g == 1:
                st["att"].probe("d", ga, o0, bar)
            o0 = o
            del o, pv, sub, bar
            d = (lambda s, res: (got[s][0, r], res)) if g == 1 else (lambda s, res: None)
            _linear(st["x1pre"], got["x1pre"][g, r], got["att"][g, r], H(g, "out_w"), H(g, "out_b"), wg, res=t[r],
                    d=d("att", t[r]))
            y, bar = ref.layernorm(got["x1pre"][g, r], H(g, "ln1_g"), H(g, "ln1_b"))
            st["x1"].check(got["x1"][g, r], y, bar, wg)
            if g == 1:
                st["x1"].probe("d", got["x1"][g, r], ref.layernorm(got["x1pre"][0, r], H(g, "ln1_g"), H(g, "ln1_b"))[0], bar)
            _linear(st["ff"], got["ff"][g, r], got["x1"][g, r], H(g, "ff1_w"), H(g, "ff1_b"), wg, relu=True,
                    d=d("x1", None))
            _linear(st["x2pre"], got["x2pre"][g, r], got["ff"][g, r], H(g, "ff2_w"), H(g, "ff2_b"), wg,
                    res=got["x1"][g, r], res_alt=got["x1pre"][g, r], d=d("ff", got["x1"][0, r] if g == 1 else None))
            ln2 = lambda s: F.layer_norm(got["x2pre"][s, r].double().view(h1 - h0, 400, 512), (512,),
                                         H(g, "ln2_g").double(), H(g, "ln2_b").double(), ref.LN_EPS)
            x2 = ln2(g)
            y, bar = ref.token_readout(x2, H(g, "fin_w"), H(g, "fin_b"))
            ho = got["head_out"][g, h0:h1]
            st["head_out"].check(ho, y, bar, wg)
            st["head_out"].probe("t", ho, ref.token_readout(x2, H(g, "fin_w"), H(g, "fin_b"), tokens=399)[0], bar)
            if g == 1:
                st["head_out"].probe("d", ho, ref.token_readout(ln2(0), H(g, "fin_w"), H(g, "fin_b"))[0], bar)
            del x2, y, bar
        del o0
    if M % 64:
        _last_tile(st["qkv"], got["qkv"], t, w["heads.in_w"], w["heads.in_b"], M)
        for g in range(2):
            _last_tile(st["x1pre"], got["x1pre"][g], got["att"][g], H(g, "out_w"), H(g, "out_b"), M, res=t)
            _last_tile(st["ff"], got["ff"][g], got["x1"][g], H(g, "ff1_w"), H(g, "ff1_b"), M, relu=True)
            _last_tile(st["x2pre"], got["x2pre"][g], got["ff"][g], H(g, "ff2_w"), H(g, "ff2_b"), M, res=got["x1"][g])
    print(f"\nrefiner N={N} ({tiles}; heads {'forked' if N <= 128 else 'serial'}):")
    bad = sum((st[s].report(f"refiner N={N}") for s in REFINE_STAGES), [])
    print(f"refiner N={N}: worst error / bar over the stages {max(s.ratio for s in st.values()):.3f}, "
          f"{time.time() - t0:.1f} s, peak torch allocation {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("N", SCORE_N)
def test_scorer_stages(setup, N):
    """Every scorer stage at N hypotheses against its float64 reference on the GPU's previous stage: qkv (bar of the
    linear layers; probes (a), (c) and, at N = 1 and 249, (f) as in test_refiner_stages), att (one group), tok_mean
    (TOKEN_BAR_U32 u32 of mean_t |att|; probe (t): the mean over 399 tokens) and feats (out_proj of the GPU's tok_mean
    in fp32, the same bar on |W| |tok_mean| + |b|; probe (c))."""
    e, W, TOK = setup
    w = W["score"]
    t0 = time.time()
    M = N * 400
    tiles = _tiles(M, (1536,), N)
    tok = TOK["score"][:N]
    got = {s: e.op_heads("score", tok, N, i) for i, s in enumerate(SCORE_STAGES)}
    t = tok.reshape(M, 512)
    st = {s: _Stage(s) for s in SCORE_STAGES}
    for h0 in range(0, N, CHUNK):
        h1 = min(N, h0 + CHUNK)
        r = slice(h0 * 400, h1 * 400)
        where = f"hypotheses {h0}..{h1 - 1}"
        _linear(st["qkv"], got["qkv"][r], t[r], w["att.in_w"], w["att.in_b"], where)
        o, pv, sub, _, _ = ref.attention(got["qkv"], N, 1, 0, h0, h1)
        st["att"].check(got["att"][r].view(h1 - h0, 400, 4, 128), o, ref.attention_bar(o, pv, sub), where)
        del o, pv, sub
        att = got["att"][r].view(h1 - h0, 400, 512)
        y, bar = ref.token_readout(att)
        st["tok_mean"].check(got["tok_mean"][h0:h1], y, bar, where)
        st["tok_mean"].probe("t", got["tok_mean"][h0:h1], ref.token_readout(att, tokens=399)[0], bar)
        tm = got["tok_mean"][h0:h1, None]
        y, bar = ref.token_readout(tm, w["att.out_w32"], w["att.out_b"])
        st["feats"].check(got["feats"][h0:h1], y, bar, where)
        st["feats"].probe("c", got["feats"][h0:h1], ref.token_readout(tm, w["att.out_w32"], ref.neighbour_panel(w["att.out_b"]))[0], bar)
    if M % 64:
        _last_tile(st["qkv"], got["qkv"], t, w["att.in_w"], w["att.in_b"], M)
    print(f"\nscorer N={N} ({tiles}):")
    bad = sum((st[s].report(f"scorer N={N}") for s in SCORE_STAGES), [])
    print(f"scorer N={N}: worst error / bar over the stages {max(s.ratio for s in st.values()):.3f}, "
          f"{time.time() - t0:.1f} s, peak torch allocation {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    assert not bad, "\n".join(bad)


def _first(out, kind, stage, N):
    """Hypotheses 0..N-1 of a stage buffer, as raw bits."""
    if kind == "refine" and 1 <= stage <= 5:
        part = out[:, :N * 400]
    elif kind == "refine" and stage == 6:
        part = out[:, :N]
    elif stage <= 1:
        part = out[:N * 400]
    else:
        part = out[:N]
    return part.view(torch.int16 if part.dtype == torch.float16 else torch.int32)


@pytest.mark.parametrize("kind", ["refine", "score"])
def test_bit_invariants(setup, kind):
    """At every stage: two launches at N = 252 are bit-equal, and hypothesis i is bit-identical across every N of the
    grid and N = 252 (identical tokens).  That spans the 128 tile against linear_ws_kernel, the eight-CTA cluster
    token reduction (N <= 66) against one CTA per sequence, and heads forked onto two streams (N <= 128) against one
    after the other: what register_objects, register_cameras and track_objects rely on to match the one-object calls."""
    e, _, TOK = setup
    grid = REFINE_N if kind == "refine" else SCORE_N
    tok = TOK[kind]
    for i, name in enumerate(REFINE_STAGES if kind == "refine" else SCORE_STAGES):
        full = e.op_heads(kind, tok, N_MAX, i)
        a = e.op_heads(kind, tok[:252], 252, i)
        b = e.op_heads(kind, tok[:252], 252, i)
        assert torch.equal(_first(a, kind, i, 252), _first(b, kind, i, 252)), f"{kind} {name}: two launches at 252 differ"
        del a, b
        for N in sorted(set(grid) | {252}):
            got = _first(e.op_heads(kind, tok[:N], N, i), kind, i, N)
            if not torch.equal(got, _first(full, kind, i, N)):
                pytest.fail(f"{kind} {name}: hypotheses 0..{N - 1} at N = {N} differ from the same hypotheses at N = {N_MAX}")
            del got
        del full
    print(f"{kind}: every stage bit-identical per hypothesis across N = {sorted(set(grid) | {252})}")


def test_refusals(setup):
    """Bad arguments are refused with an error before anything is enqueued: no kernel launch is counted."""
    import ctypes as C

    from foundationpose_b200 import _lib
    from foundationpose_b200.engine import Engine, _stream

    e, _, TOK = setup
    tok = TOK["refine"][:1]
    out = torch.empty(400, 3072, dtype=torch.float16, device="cuda")
    host = torch.empty(400, 3072, dtype=torch.float16)
    host_tok = tok.cpu()
    p = lambda x: C.c_void_p(x.data_ptr())
    fresh = Engine()
    cases = {
        "which = 2": (e._h, 2, p(tok), 1, 0, p(out)),
        "which = -1": (e._h, -1, p(tok), 1, 0, p(out)),
        "stage = -1": (e._h, 0, p(tok), 1, -1, p(out)),
        "refiner stage = 7": (e._h, 0, p(tok), 1, 7, p(out)),
        "scorer stage = 4": (e._h, 1, p(tok), 1, 4, p(out)),
        "N = 0": (e._h, 0, p(tok), 0, 0, p(out)),
        "N = 513": (e._h, 0, p(tok), 513, 0, p(out)),
        "null tok": (e._h, 0, None, 1, 0, p(out)),
        "null out": (e._h, 0, p(tok), 1, 0, None),
        "host out": (e._h, 0, p(tok), 1, 0, p(host)),
        "host tok": (e._h, 0, p(host_tok), 1, 0, p(out)),
        "null context": (None, 0, p(tok), 1, 0, p(out)),
        "weights not loaded": (fresh._h, 0, p(tok), 1, 0, p(out)),
    }
    torch.cuda.synchronize()
    for what, args in cases.items():
        before = _lib.launch_count()
        rc = _lib.lib.fp_op_heads(*args, _stream())
        assert rc < 0, f"{what}: accepted (rc {rc})"
        assert _lib.launch_count() == before, f"{what}: refused after launching kernels"
    fresh.close()
    with pytest.raises(ValueError):
        e.op_heads("refine", tok, 1, 7)
