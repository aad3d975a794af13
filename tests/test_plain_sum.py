"""Plaintext matrix x ciphertext vector: b200_plain_to_ntt, b200_multiply_plain_sum and B200_Evaluator_MultiplyPlainSum
against the reference's multiply_plain + add_inplace chain, word for word.  The same checks run on the CPU emulation build
and, marked gpu, on the CUDA library."""
import ctypes as C

import numpy as np
import pytest

import parity_checks as pc
from backends import CudaBackend, EmuBackend
from params import PARAMS, PLAIN_EDGE
from refseal import COR_E_INVALIDOPERATION, E_INVALIDARG, E_POINTER, SealError
from sealc_driver import Sealc
from sunscreen_b200.lib import PLAIN_NTT_MULTIPLY, PLAIN_NTT_TRANSFORM

vp, u64 = C.c_void_p, C.c_uint64

EMU_SETS = ["n4096", "n8192", "n4096_q_below_t"] + [p for p in PLAIN_EDGE if PARAMS[p][0] <= 8192]
CHAIN_SETS = ["n4096", "n8192", "n8192_49", "n8192_54", "n8192_60", "n4096_q_below_t"]


def signed_plain(v, t):
    """Sunscreen's `Signed` encoding: bit i of |v| at x^i, as 1 or (for v < 0) t - 1 (sunscreen/src/types/bfv/signed.rs)."""
    a = abs(v)
    return np.array([((a >> i) & 1) * (t - 1 if v < 0 else 1) for i in range(max(a.bit_length(), 1))], dtype=np.uint64)


def padded(p, n):
    out = np.zeros(n, dtype=np.uint64)
    out[: p.size] = p
    return out


def operand_plains(n, t, rng):
    """Every plain_operand_classes plaintext and the Signed encodings of +-1, +-4, +-5 and -123, shuffled."""
    out = [c[1] for c in pc.plain_operand_classes(n, t, rng)]
    out += [padded(signed_plain(v, t), n) for v in (1, -1, 4, -4, 5, -5, -123)]
    return [out[i] for i in rng.permutation(len(out))]


def data_levels(P):
    """(layer-1 level, reference data level index, k) of every data level"""
    out = []
    for j in range(len(P.ref.data_parms_ids())):
        lv = P.ctx.first_level + j
        out.append((lv, j, P.ctx.level_info(lv)["k"]))
    return out


def ref_transform_to_ntt(P, coeffs, j):
    """Evaluator::transform_to_ntt(Plaintext, parms_id) of the reference: NTT-form words [k][n] at data level j"""
    R = P.ref
    pt, dst = R.new_pt(coeffs), vp()
    R.ref.call("Plaintext_Create1", None, C.byref(dst))
    R.ref.call("Evaluator_TransformToNTT1", R.ev, pt, R.data_parms_ids()[j], dst, None)
    words = R.pt_coeffs(dst)
    R.free_pt(pt)
    R.free_pt(dst)
    return words.reshape(-1, P.n)


def ref_chain(P, cts, plains, j):
    """[R][size][k][n] words of multiply_plain(ct_0, p_i0) + ... + multiply_plain(ct_{m-1}, p_i,m-1), the reference's chain.
    A product the reference refuses as transparent contributes nothing (layer 1 returns zeros for it)."""
    R = P.ref
    rcts = [R.new_ct(c, level=j) for c in cts]
    rows = []
    for prow in plains:
        acc = None
        for ct, p in zip(rcts, prow):
            rp = R.new_pt(p)
            try:
                prod = R.multiply_plain(ct, rp)
            except SealError as e:
                assert e.code == COR_E_INVALIDOPERATION, e
                continue
            finally:
                R.free_pt(rp)
            if acc is None:
                acc = prod
            else:
                nxt = R.add(acc, prod)
                R.free_ct(acc)
                R.free_ct(prod)
                acc = nxt
        rows.append(np.zeros(cts[0].shape, dtype=np.uint64) if acc is None else R.ct_words(acc))
        if acc is not None:
            R.free_ct(acc)
    for h in rcts:
        R.free_ct(h)
    return np.stack(rows)


def plain_sum(P, cts, plains, lv, rule=PLAIN_NTT_MULTIPLY, plain_ntt=None):
    """b200_plain_to_ntt(rule) of `plains` [R][m][n] (or the given NTT-form words), then b200_multiply_plain_sum"""
    m, size, k, n = cts.shape
    R = len(plains) if plain_ntt is None else plain_ntt.shape[0]
    if plain_ntt is None:
        pn = P.out(R, m, k, n)
        P.ctx.plain_to_ntt(P.dev(np.asarray(plains).reshape(R * m, n)), R * m, pn, rule=rule, level=lv)
    else:
        pn = P.dev(plain_ntt)
    out = P.out(R, size, k, n)
    P.ctx.multiply_plain_sum(P.dev(cts), size, m, pn, R, out, level=lv)
    return P.host(out).reshape(R, size, k, n)


# ---- the checks, shared by both backends ----

def check_transform_rule(P, seed=5):
    """b200_plain_to_ntt(TRANSFORM) == the reference's TransformToNTT1 for every class with coefficients below t (the reference
    validates the values there), at every data level"""
    rng = np.random.default_rng(seed)
    plains = [p for p in operand_plains(P.n, P.t, rng) if int(p.max()) < P.t]
    B = len(plains)
    d = P.dev(np.stack(plains))
    for lv, j, k in data_levels(P):
        out = P.out(B, k, P.n)
        P.ctx.plain_to_ntt(d, B, out, rule=PLAIN_NTT_TRANSFORM, level=lv)
        got = P.host(out).reshape(B, k, P.n)
        for i, p in enumerate(plains):
            pc.eq(got[i], ref_transform_to_ntt(P, p, j), f"plain_to_ntt(TRANSFORM) level {lv} item {i}")


def check_coefficient_chain(P, R=3, m=5, seed=7):
    """coefficient-form plaintexts (MULTIPLY rule) summed by b200_multiply_plain_sum == the reference's chain, every class in
    some R x m matrix, at every data level"""
    rng = np.random.default_rng(seed)
    plains = operand_plains(P.n, P.t, rng)
    mats = -(-len(plains) // (R * m))
    plains = (plains * 2)[: mats * R * m]
    for lv, j, k in data_levels(P):
        for a in range(mats):
            mat = np.stack(plains[a * R * m:(a + 1) * R * m]).reshape(R, m, P.n)
            cts = pc.rand_ct(rng, P.moduli[:k], k, P.n, batch=m)
            pc.eq(plain_sum(P, cts, mat, lv), ref_chain(P, cts, mat, j), f"plain sum level {lv} matrix {a}")


def check_ntt_chain(P, seed=9):
    """NTT-form plaintexts made by the reference's TransformToNTT1 == its TransformToNTT2 -> multiply_plain -> add ->
    TransformFromNTT chain.  With an upper-half monomial in the matrix the two lifts differ (under the fast plain lift), and
    each result matches its own chain."""
    rng = np.random.default_rng(seed)
    Rr = P.ref
    lv, j, k = data_levels(P)[0]
    m = 3
    thr = (P.t + 1) // 2
    mono = np.zeros(P.n, dtype=np.uint64)
    mono[1] = P.t - 1
    mat = [[mono, rng.integers(0, P.t, P.n, dtype=np.uint64), padded(signed_plain(-5, P.t), P.n)],
           [rng.integers(thr, P.t, P.n, dtype=np.uint64), mono, padded(signed_plain(3, P.t), P.n)]]
    cts = pc.rand_ct(rng, P.moduli[:k], k, P.n, batch=m)
    pn = np.stack([np.stack([ref_transform_to_ntt(P, p, j) for p in row]) for row in mat])
    got_ntt = plain_sum(P, cts, None, lv, plain_ntt=pn)
    # the reference's NTT-form chain
    exp = []
    rcts = []
    for c in cts:
        h, d = Rr.new_ct(c, level=j), Rr.new_ct()
        Rr.ref.call("Evaluator_TransformToNTT2", Rr.ev, h, d)
        Rr.free_ct(h)
        rcts.append(d)
    for i, row in enumerate(mat):
        acc = None
        for jj, p in enumerate(row):
            rp, dst = Rr.new_pt(p), vp()
            Rr.ref.call("Plaintext_Create1", None, C.byref(dst))
            Rr.ref.call("Evaluator_TransformToNTT1", Rr.ev, rp, Rr.data_parms_ids()[j], dst, None)
            prod = Rr.multiply_plain(rcts[jj], dst)
            Rr.free_pt(rp)
            Rr.free_pt(dst)
            acc = prod if acc is None else Rr.add(acc, prod)
        out = Rr.new_ct()
        Rr.ref.call("Evaluator_TransformFromNTT", Rr.ev, acc, out)
        exp.append(Rr.ct_words(out))
    pc.eq(got_ntt, np.stack(exp), "NTT-form plaintext chain")
    got_coeff = plain_sum(P, cts, mat, lv)
    pc.eq(got_coeff, ref_chain(P, cts, mat, j), "coefficient plaintext chain")
    if all(q > P.t for q in P.moduli[:k]):
        assert not np.array_equal(got_coeff, got_ntt), "the upper-half monomial should separate the two lifts"


def check_exact_accumulation(P, m=300):
    """every NTT-domain word of X and P equal to q - 1: each output word is m (q-1)^2 = m mod q in the NTT domain, past the
    integer path's 256-term bound and the FP64 path's 16-term one"""
    lv, j, k = data_levels(P)[0]
    qs = P.moduli[:k]
    qm1 = np.array(qs, dtype=np.uint64)[:, None] - np.uint64(1)
    one = np.stack([P.ref.ref.ntt_inverse(q, np.full(P.n, q - 1, dtype=np.uint64)) for q in qs])
    cts = np.broadcast_to(one, (m, 2, k, P.n)).copy()
    pn = np.broadcast_to(qm1, (1, m, k, P.n)).copy()
    got = plain_sum(P, cts, None, lv, plain_ntt=pn)
    exp = np.stack([P.ref.ref.ntt_inverse(q, np.full(P.n, m % q, dtype=np.uint64)) for q in qs])
    pc.eq(got, np.broadcast_to(exp, got.shape), f"sum of {m} (q-1)^2 terms")


def sealc_chain(S, ref, name, rows=3, cols=4, seed=11, monkeypatch=None):
    """B200_Evaluator_MultiplyPlainSum through the SEAL-named layer == the reference chain's words; the error HRESULTs; a
    destination that aliases an operand; and (with a scratch bound of one row) the row chunking"""
    from refseal import RefContext
    n, moduli, t = PARAMS[name]
    Rr = RefContext(n, moduli, t)
    ctx = S.context(n, moduli, t)
    k = ctx.k
    rng = np.random.default_rng(seed)
    plains = operand_plains(n, t, rng)
    plains = [p for p in plains if p.any()]
    mat = [[plains[(i * cols + jj) % len(plains)] for jj in range(cols)] for i in range(rows)]
    cts = pc.rand_ct(rng, moduli[:k], k, n, batch=cols)
    Pfake = type("P", (), {"ref": Rr, "n": n})()
    exp = ref_chain(Pfake, cts, mat, 0)

    def run(enc_h, pl_h, dst_h, r=rows, c=cols, ev=ctx.ev):
        return S.rc("B200_Evaluator_MultiplyPlainSum", ev, u64(r), u64(c), (vp * len(enc_h))(*enc_h) if enc_h is not None else None,
                    (vp * len(pl_h))(*pl_h) if pl_h is not None else None, (vp * len(dst_h))(*dst_h) if dst_h is not None else None)

    enc_h = [ctx.new_ct(c) for c in cts]
    pl_h = [ctx.new_pt(p) for row in mat for p in row]
    dst_h = [ctx._dst() for _ in range(rows)]
    assert run(enc_h, pl_h, dst_h) == 0
    for i in range(rows):
        pc.eq(ctx.ct_words(dst_h[i]), exp[i], f"{name}: MultiplyPlainSum row {i}")
    # chunked over rows: a scratch bound of one row's NTT-form plaintexts
    if monkeypatch is not None:
        monkeypatch.setenv("B200_PLAIN_SUM_SCRATCH", str(cols * k * n * 8))
        dst2 = [ctx._dst() for _ in range(rows)]
        assert run(enc_h, pl_h, dst2) == 0
        for i in range(rows):
            pc.eq(ctx.ct_words(dst2[i]), exp[i], f"{name}: chunked MultiplyPlainSum row {i}")
        monkeypatch.delenv("B200_PLAIN_SUM_SCRATCH")
    # a destination aliasing an operand: every operand is read before the first write
    alias = [ctx.new_ct(c) for c in cts]
    assert run(alias, pl_h, [alias[1]] + [ctx._dst() for _ in range(rows - 1)]) == 0
    pc.eq(ctx.ct_words(alias[1]), exp[0], f"{name}: destination aliasing encrypteds[1]")
    # errors, each against the reference chain's HRESULT where the chain has one
    zero = ctx.new_pt(np.zeros(1, dtype=np.uint64))
    bad_pl = list(pl_h)
    bad_pl[cols + 1] = zero
    assert run(enc_h, bad_pl, dst_h) == COR_E_INVALIDOPERATION
    rz = Rr.new_pt(np.zeros(1, dtype=np.uint64))
    with pytest.raises(SealError) as e:
        Rr.multiply_plain(Rr.new_ct(cts[0]), rz)
    assert e.value.code == COR_E_INVALIDOPERATION
    ntt_ct = ctx.new_ct(cts[0], ntt=True)
    assert run([enc_h[0], ntt_ct] + enc_h[2:], pl_h, dst_h) == E_INVALIDARG
    if len(Rr.data_parms_ids()) > 1:
        low = ctx.mod_switch_to_next(enc_h[0])
        assert run(enc_h[:-1] + [low], pl_h, dst_h) == E_INVALIDARG
    size3 = ctx.new_ct(np.concatenate([cts[0], cts[1][:1]]))
    assert run([size3] + enc_h[1:], pl_h, dst_h) == E_INVALIDARG
    assert run(enc_h, pl_h, dst_h, ev=None) == E_POINTER
    assert run(None, pl_h, dst_h) == E_POINTER
    assert run(enc_h, pl_h, [None] + dst_h[1:]) == E_INVALIDARG
    assert run(enc_h, pl_h, dst_h, c=0) == E_INVALIDARG
    assert run(enc_h, pl_h, dst_h, r=0) == 0
    # a transparent final result (polys 1.. all zero), which the chain's first multiply_plain already refuses
    tr = cts.copy()
    tr[:, 1] = 0
    tr_h = [ctx.new_ct(c) for c in tr]
    assert run(tr_h, pl_h, dst_h) == COR_E_INVALIDOPERATION
    with pytest.raises(SealError) as e:
        Rr.multiply_plain(Rr.new_ct(tr[0]), Rr.new_pt(mat[0][0]))
    assert e.value.code == COR_E_INVALIDOPERATION
    # size-3 operands throughout
    c3 = pc.rand_ct(rng, moduli[:k], k, n, size=3, batch=cols)
    h3 = [ctx.new_ct(c) for c in c3]
    d3 = [ctx._dst() for _ in range(rows)]
    assert run(h3, pl_h, d3) == 0
    exp3 = ref_chain(Pfake, c3, mat, 0)
    for i in range(rows):
        pc.eq(ctx.ct_words(d3[i]), exp3[i], f"{name}: size-3 MultiplyPlainSum row {i}")


# ---- CPU emulation build ----

@pytest.fixture(scope="module", params=EMU_SETS)
def emu_pair(request, emu_lib, ref):
    return pc.pair_for(EmuBackend(emu_lib), request.param)


def test_plain_to_ntt_transform_rule(emu_pair):
    check_transform_rule(emu_pair)


@pytest.mark.parametrize("name", CHAIN_SETS + [p for p in PLAIN_EDGE if PARAMS[p][0] <= 8192])
def test_coefficient_plaintext_chain(emu_lib, ref, name):
    check_coefficient_chain(pc.pair_for(EmuBackend(emu_lib), name))


@pytest.mark.parametrize("name", ["n4096", "n8192", "n4096_q_below_t"])
def test_ntt_form_plaintext_chain(emu_lib, ref, name):
    check_ntt_chain(pc.pair_for(EmuBackend(emu_lib), name))


@pytest.mark.parametrize("name", ["n8192_60", "n8192_49"])
def test_exact_accumulation(emu_lib, ref, name):
    check_exact_accumulation(pc.pair_for(EmuBackend(emu_lib), name))


@pytest.mark.parametrize("name", ["n4096", "n4096_q_below_t"])
def test_sealc_multiply_plain_sum(emu_lib, ref, name, monkeypatch):
    sealc_chain(Sealc(emu_lib.lib), ref, name, monkeypatch=monkeypatch)


def test_layer1_arguments(emu_lib):
    from sunscreen_b200.lib import B200Context, B200Error
    n, moduli, t = PARAMS["n4096"]
    ctx = B200Context(n, moduli, t, lib=emu_lib)
    k = ctx.k()
    buf = np.zeros((4, 2, k, n), dtype=np.uint64)
    with pytest.raises(B200Error) as e:
        ctx.multiply_plain_sum(buf, 2, 2, None, 1, buf[2:])
    assert e.value.code == -4
    with pytest.raises(B200Error) as e:
        ctx.multiply_plain_sum(buf, 0, 2, buf, 1, buf[2:])
    assert e.value.code == -1
    with pytest.raises(B200Error) as e:  # out overlapping cts
        ctx.multiply_plain_sum(buf, 2, 2, buf[2:], 1, buf[1:])
    assert e.value.code == -1
    with pytest.raises(B200Error) as e:
        ctx.plain_to_ntt(buf, 1, buf[1:], rule=2)
    assert e.value.code == -1
    ctx.multiply_plain_sum(buf, 2, 0, buf, 1, buf[2:])
    ctx.multiply_plain_sum(buf, 2, 2, buf, 0, buf[2:])
    ctx.plain_to_ntt(buf, 0, buf[1:])


# ---- CUDA library ----

@pytest.fixture(scope="module")
def cuda_be():
    return CudaBackend()


@pytest.mark.gpu
@pytest.mark.parametrize("name", EMU_SETS)
def test_gpu_plain_to_ntt_transform_rule(cuda_be, ref, name):
    check_transform_rule(pc.pair_for(cuda_be, name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CHAIN_SETS + PLAIN_EDGE)
def test_gpu_coefficient_plaintext_chain(cuda_be, ref, name):
    check_coefficient_chain(pc.pair_for(cuda_be, name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n4096", "n8192", "n4096_q_below_t"])
def test_gpu_ntt_form_plaintext_chain(cuda_be, ref, name):
    check_ntt_chain(pc.pair_for(cuda_be, name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192_60", "n8192_49"])
def test_gpu_exact_accumulation(cuda_be, ref, name):
    check_exact_accumulation(pc.pair_for(cuda_be, name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192_60", "n8192_49", "n8192"])
def test_gpu_long_sums_match_multiply_plain_and_add(cuda_be, name):
    """m = 300 random terms against b200_multiply_plain + b200_add on the same device, at R = 2 and size 2"""
    from sunscreen_b200.lib import B200Context
    n, moduli, t = PARAMS[name]
    ctx = B200Context(n, moduli, t)
    k = ctx.k()
    rng = np.random.default_rng(3)
    m, R = 300, 2
    P = type("P", (), {"ctx": ctx, "dev": staticmethod(cuda_be.to_dev), "out": staticmethod(lambda *s: cuda_be.empty(s)),
                       "host": staticmethod(cuda_be.to_host)})()
    cts = pc.rand_ct(rng, moduli[:k], k, n, batch=m)
    plains = rng.integers(0, t, size=(R, m, n), dtype=np.uint64)
    got = plain_sum(P, cts, plains, None)
    dc = cuda_be.to_dev(cts)
    for i in range(R):
        prod = cuda_be.empty((m, 2, k, n))
        ctx.multiply_plain(dc, 2, cuda_be.to_dev(plains[i]), m, prod, m)
        acc = prod[0].clone()
        for j in range(1, m):
            ctx.add(acc, prod[j], acc, 2, 1)
        pc.eq(got[i], cuda_be.to_host(acc), f"{name}: row {i} of 300-term sums")


@pytest.mark.gpu
def test_gpu_shapes(cuda_be, ref):
    """R = m = 1 (== b200_multiply_plain), size 3, output row counts on both sides of the NTT's 256/512-thread switch, and
    n = 32768 at R = m = 2, against the reference"""
    P = pc.pair_for(cuda_be, "n8192")
    rng = np.random.default_rng(13)
    lv, j, k = data_levels(P)[0]
    # R = m = 1
    ct = pc.rand_ct(rng, P.moduli[:k], k, P.n, batch=1)
    p = rng.integers(0, P.t, size=(1, 1, P.n), dtype=np.uint64)
    o = P.out(1, 2, k, P.n)
    P.ctx.multiply_plain(P.dev(ct), 2, P.dev(p[0]), 1, o, 1)
    pc.eq(plain_sum(P, ct, p, lv), P.host(o), "R = m = 1 vs multiply_plain")
    # size 3 (one output row: the 512-thread NTT) and many rows (the 256-thread NTT)
    for R, m in ((1, 4), (2 * P.ctx.sm_count, 2)):
        c3 = pc.rand_ct(rng, P.moduli[:k], k, P.n, size=3, batch=m)
        mat = [[rng.integers(0, P.t, P.n, dtype=np.uint64) for _ in range(m)] for _ in range(R)]
        got = plain_sum(P, c3, np.array(mat), lv)
        if R <= 4:
            pc.eq(got, ref_chain(P, c3, mat, j), f"size 3, R = {R}, m = {m}")
        else:
            # rows against the reference at both ends of the batch
            sel = [0, R - 1]
            pc.eq(got[sel], ref_chain(P, c3, [mat[i] for i in sel], j), f"size 3, R = {R}, m = {m}")
    P32 = pc.pair_for(cuda_be, "n32768")
    lv, j, k = data_levels(P32)[0]
    cts = pc.rand_ct(rng, P32.moduli[:k], k, P32.n, batch=2)
    mat = [[rng.integers(0, P32.t, P32.n, dtype=np.uint64) for _ in range(2)] for _ in range(2)]
    pc.eq(plain_sum(P32, cts, np.array(mat), lv), ref_chain(P32, cts, mat, j), "n32768, R = m = 2")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n4096", "n8192", "n4096_q_below_t"])
def test_gpu_sealc_multiply_plain_sum(cuda_be, ref, name, monkeypatch):
    sealc_chain(Sealc(cuda_be.lib.lib), ref, name, monkeypatch=monkeypatch)
