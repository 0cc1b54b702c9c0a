"""GPU tests of the whole training step under dropout: ``forward(encoder=..., decoder=...)`` (modules/model.py FusedT5EncodeTrain,
FusedT5DecodeTrain, the heads and the loss) and its backward against the float64 statement of tests/t5_enc_train_ref.py and
tests/t5_dec_train_ref.py, run with the pass's own dropout and relu decisions.

The pass's decisions are taken from the pass itself, in HF's call order:
  * token-wise dropout sites: ``modules.model.dropout_rows`` applies the next mask of an HF-order list (``random_masks``), the
    kept rows of an encoder mask, the first T positions of a decoder mask; HF's halves of a mixed pass draw from the same list
    through a patched ``F.dropout``;
  * attention-weight sites: the seeds the pass draws through ``ops.t5enc_dropout_seed`` are recorded, and the keep bits
    ``ops.t5enc_dropout_keep`` exports for them replace those sites' entries of the list;
  * relu: ``pre > 0`` at every feed-forward relu (``F.relu`` catches both ``_train_feed_forward`` and HF's ``nn.ReLU``).
The statement then runs on a float64 copy of the model with those masks, so the pass and the statement differ by rounding only.
A relu audit compares the pass's relu decisions with the statement's float64 signs, and negative controls show that a dropout
site in the wrong layer, a missing 1/(1 - p) or cross-attention bits read at the packed row instead of the encoder position
exceed the bounds tenfold.  `pytest -m gpu`."""
import copy

import numpy as np
import pytest
import torch

import t5_dec_train_ref as DR
import t5_enc_ref as E
import t5_enc_train_ref as TR
from test_gpu_decode import highest
from test_gpu_decode_train import keep_bits
from test_gpu_encode_tc import high
from test_gpu_encode_train import amazon, set_dropout, train_batch
from test_t5_dec_train_ref import batch_of
from test_t5_enc_ref import inputs, random_model

pytestmark = pytest.mark.gpu

#: arm -> (encoder, decoder, encoder_attention, through torch.compile)
ARMS = {"fused/fused": ("fused", "fused", "fp32", False), "fused/fused tf32": ("fused", "fused", "tf32", False),
        "fused/hf": ("fused", "hf", "fp32", False), "hf/fused": ("hf", "fused", "fp32", False),
        "fused/fused compiled": ("fused", "fused", "fp32", True)}
# Bounds, from every case of this file on an H100 80GB HBM3 (700 W), worst measured in brackets:
#: fp32 arms: the loss's relative error [1.5e-7] and each gradient's error relative to its parameter's largest entry [3.8e-6]
LOSS_BOUND = 1e-6
GRAD_BOUND = 3e-5
#: TF32 arm: each gradient at most TF32_FACTOR times the error of the float32 statement under TF32 matmuls, floored at
#: TF32_FLOOR of the largest entry [1.02 times]; the loss within TF32_LOSS_BOUND relative [3.2e-5]
TF32_FACTOR, TF32_FLOOR, TF32_LOSS_BOUND = 4, 2 * 2 ** -11, 2e-4
#: relu audit: every decision the pass and the float64 statement disagree on sits within this many fp32 units (2^-24) of its
#: site's largest |pre-activation| [2.1; with the TF32 attention, 1923]
RELU_ULPS = {"fp32": 16, "tf32": 2 ** 14}


class Layout:
    """The encoder layout of a batch: B, S, T, the kept positions' flat index src (b * S + p) and the masks' split."""

    def __init__(self, m, batch):
        from rq_vae_recommender_b200.modules import model as M
        H = self.T = m.num_hierarchies
        self.mask = M._strip_dedup_col(batch.seq_mask.long(), H + 1, H)
        self.ids = M._strip_dedup_col(batch.sem_ids, H + 1, H)
        self.fut = batch.sem_ids_fut[:, :H]
        self.sep, self.user = m.sep_token is not None, m.user_embedding is not None
        keep, _ = E.kept_positions(self.mask, H, self.sep, self.user)
        self.B, self.S = keep.shape
        assert self.S != H + 1                                      # a decoder site's shape tells self- from cross-attention
        self.src = keep.reshape(-1).nonzero().squeeze(1)
        self.n_enc = len(TR.dropout_shapes(m, self.B, self.S))
        self.layers = m.encoder.config.num_layers

    def random_masks(self, m, p, seed):
        dev = self.mask.device
        return ([k.to(dev) for k in TR.random_masks(m, self.B, self.S, p, seed, torch.bool)]
                + [k.to(dev) for k in DR.random_masks(m, self.B, self.T, self.S, p, seed + 1, torch.bool)])

    def rows(self, i, mask):
        """The rows of HF-order site i's [B, *, w] mask that the fused pass's [rows, w] tensor at that site holds."""
        w = mask.shape[-1]
        return mask.reshape(self.B * self.S, w)[self.src] if i < self.n_enc else mask[:, :self.T].reshape(self.B * self.T, w)

    def relu_rows(self, j, mask):
        return self.rows(0 if j < self.layers else self.n_enc, mask)


def run_pass(m, batch, arm, masks, p, fn=None):
    """forward + backward of ``arm`` with the dropout masks ``masks`` (HF order; None in eval mode): (loss, {name: grad},
    the masks the pass applied with its attention sites' keep bits in place, its relu decisions at HF's shapes)."""
    import torch.nn.functional as F
    from rq_vae_recommender_b200 import ops
    from rq_vae_recommender_b200.modules import model as M
    encoder, decoder, attention, _ = ARMS[arm]
    lay = Layout(m, batch)
    B, S, T = lay.B, lay.S, lay.T
    used = list(masks) if masks is not None else []
    taken, seeds, relus = [0], [], []

    def take(x_dims):
        i = taken[0]
        taken[0] += 1
        assert used[i].dim() == x_dims, (i, used[i].shape)
        return i, used[i]

    def rows_dropout(x, q):
        if q == 0:
            return x
        assert q == p
        i, mk = take(3)
        mk = lay.rows(i, mk)
        assert x.shape == mk.shape, (i, x.shape, mk.shape)
        return x * mk.to(x.dtype) / (1 - q)

    def hf_dropout(x, p=0.5, training=True, inplace=False):
        if not training:
            return x
        i, mk = take(x.dim())
        assert mk.shape == x.shape, (i, mk.shape, x.shape)
        return x * mk.to(x.dtype) / (1 - p)

    def seed(device):
        s = real_seed(device)
        i, _ = take(4)
        seeds.append((i, s.clone()))
        return s

    def relu(x, inplace=False):
        relus.append(x.detach() > 0)
        return real_relu(x, inplace=inplace)

    real_rows, real_dropout, real_seed, real_relu = M.dropout_rows, F.dropout, ops.t5enc_dropout_seed, F.relu
    M.dropout_rows, F.dropout, ops.t5enc_dropout_seed, F.relu = rows_dropout, hf_dropout, seed, relu
    try:
        with highest():
            m.zero_grad(set_to_none=True)
            loss = (m if fn is None else fn)(batch, encoder=encoder, decoder=decoder, encoder_attention=attention).loss
            loss.backward()
    finally:
        M.dropout_rows, F.dropout, ops.t5enc_dropout_seed, F.relu = real_rows, real_dropout, real_seed, real_relu
    assert taken[0] == len(used)                                    # every site consumed its mask, none more
    for i, s in seeds:
        shape = used[i].shape
        heads = shape[1]
        if i < lay.n_enc:
            assert shape == (B, heads, S, S)
            used[i] = ops.t5enc_dropout_keep(s, p, B, heads, S).bool()
        else:
            bits = keep_bits(s, p, B, heads, T, shape[3] if shape[3] == S else T).bool()
            used[i] = torch.zeros(shape, dtype=torch.bool, device=bits.device)
            used[i][:, :, :T, :bits.shape[3]] = bits
    assert len(relus) == 2 * lay.layers
    hf_relus = []
    for j, r in enumerate(relus):
        if r.dim() == 3:                                            # HF's own feed-forward: already [B, positions, d_ff]
            hf_relus.append(r)
        elif j < lay.layers:
            full = torch.zeros((B * S, r.shape[1]), dtype=torch.bool, device=r.device)
            full[lay.src] = r
            hf_relus.append(full.view(B, S, -1))
        else:
            hf_relus.append(torch.cat([r.view(B, T, -1), r.new_zeros(B, 1, r.shape[1])], dim=1))
    grads = {n: prm.grad.clone() for n, prm in m.named_parameters() if prm.grad is not None}
    return loss.detach(), grads, (used if masks is not None else None), hf_relus


def statement(mx, batch, masks, relus, p, pre=None, packed_row_bits=False):
    """The float64 (or float32) statement's loss on model copy mx under the given masks and relu decisions.  packed_row_bits
    reads the cross-attention keep bits at each key's packed row instead of its encoder position (a negative control)."""
    lay = Layout(mx, batch)
    L = lay.layers
    enc_masks, dec_masks = (masks[:lay.n_enc], masks[lay.n_enc:]) if masks is not None else (None, None)
    enc_relus, dec_relus = (relus[:L], relus[L:]) if relus is not None else (None, None)
    out, _ = TR.encode_train(mx, lay.mask, lay.ids, batch.user_ids, enc_masks, p, enc_relus, pre)
    rows, offs, key_mask, kpos = DR.packed_layout(out, lay.mask, lay.T, lay.sep, lay.user)
    if packed_row_bits:
        counts = (offs[1:] - offs[:-1]).long()
        kpos = torch.arange(rows.shape[0], device=rows.device) - torch.repeat_interleave(offs[:-1].long(), counts)
    dec = DR.decode_train(mx, lay.fut, rows, offs, key_mask, kpos, dec_masks, p, dec_relus, pre)
    return DR.level_loss(mx, dec, lay.fut)


def statement_grads(mx, batch, masks, relus, p, **kw):
    mx.zero_grad(set_to_none=True)
    loss = statement(mx, batch, masks, relus, p, **kw)
    loss.backward()
    return loss.detach(), {n: prm.grad for n, prm in mx.named_parameters() if prm.grad is not None}


def grad_errors(got, want):
    """{name: max |got - want| / max |want|} over every parameter either side has a gradient for."""
    errs = {}
    for name in set(got) | set(want):
        w = want[name].double() if name in want else torch.zeros_like(got[name], dtype=torch.float64)
        g = got[name].double() if name in got else torch.zeros_like(w)
        top = w.abs().max().item()
        diff = (g - w).abs().max().item()
        errs[name] = diff / top if top > 0 else (0.0 if diff == 0 else float("inf"))
    return errs


def relu_audit(lay, relus, pre, ulps):
    """(disagreements, the largest |pre64| among them in fp32 units of its site's largest |pre64|) of the pass's relu decisions
    against the float64 statement's signs; asserts that every disagreement sits within ``ulps`` units."""
    count, worst = 0, 0.0
    for j, (r, x) in enumerate(zip(relus, pre)):
        bad = lay.relu_rows(j, r) != (x > 0)
        n = int(bad.sum())
        if n:
            units = (x[bad].abs().max() / (x.abs().max() * 2 ** -24)).item()
            assert units <= ulps, (j, n, units)
            count, worst = count + n, max(worst, units)
    return count, worst


def check_arm(m, batch, arm, p, masks, label, fn=None):
    """One arm against the float64 statement, printing the errors and the relu audit: (the masks the pass applied, its relu
    decisions, its gradients, the relu disagreements)."""
    lay = Layout(m, batch)
    loss, grads, used, relus = run_pass(m, batch, arm, masks, p, fn)
    m64 = copy.deepcopy(m).double()
    pre = []
    loss64, g64 = statement_grads(m64, batch, used, relus, p, pre=pre)
    tf32 = ARMS[arm][2] == "tf32"
    flips, units = relu_audit(lay, relus, pre, RELU_ULPS["tf32" if tf32 else "fp32"])
    loss_err = abs(loss.item() - loss64.item()) / max(abs(loss64.item()), 1e-30)
    errs = grad_errors(grads, g64)
    worst = max(errs, key=errs.get)
    print(f"{label} [{arm}]: loss {loss_err:.2e}, largest gradient error {errs[worst]:.2e} of the largest entry ({worst}), "
          f"relu disagreements {flips} (largest |pre| {units:.1f} fp32 units)")
    if not tf32:
        assert loss_err <= LOSS_BOUND, (label, arm, loss_err)
        for name, err in errs.items():
            assert err <= GRAD_BOUND, (label, arm, name, err)
        return used, relus, grads, flips
    # the same statement in float32 under TF32 matmuls, with the same masks and relu decisions
    with high():
        loss32, g32 = statement_grads(copy.deepcopy(m), batch, used, relus, p)
    cmp = grad_errors(g32, g64)
    cmp_loss = abs(loss32.item() - loss64.item()) / max(abs(loss64.item()), 1e-30)
    assert loss_err <= TF32_LOSS_BOUND, (label, arm, loss_err, cmp_loss)
    for name, err in errs.items():
        assert err <= max(TF32_FACTOR * cmp[name], TF32_FLOOR), (label, arm, name, err, cmp[name])
    print(f"{label} [{arm}]: largest ratio to the TF32-matmul statement "
          f"{max(errs[n] / max(cmp[n], TF32_FLOOR) for n in errs):.2f}, loss {loss_err:.2e} against its {cmp_loss:.2e}")
    return used, relus, grads, flips


def check_case(m, batch, p, label, arms=tuple(ARMS), seed=0):
    masks = Layout(m, batch).random_masks(m, p, seed) if m.training else None
    for arm in arms:
        fn = None
        if ARMS[arm][3]:
            torch._dynamo.reset()
            fn = torch.compile(m)
        check_arm(m, batch, arm, p, masks, label, fn)


def cuda_batch(batch):
    return type(batch)(*(t.cuda() for t in batch))


# ------------------------------------------------------------------------------------------------ cases
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_amazon_shape(mode):
    """configs/decoder_amazon.gin's shape: 64 histories of 1 to 20 items, p = 0.1; in eval mode no dropout site fires."""
    rs = np.random.RandomState(3)
    m = amazon()
    set_dropout(m, 0.1)
    m.train(mode == "train")
    batch = train_batch(rs, 64, 20, 3, 256, rs.randint(1, 21, size=64))
    check_case(m, batch, 0.1, f"amazon {mode}")


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("kind", ["full", "end", "holes", "empty"])
@pytest.mark.parametrize("H", [3, 5, 8])
@pytest.mark.parametrize("sep,user_bins", [(True, None), (False, None), (True, 7), (False, 7)])
def test_small_model(sep, user_bins, H, kind, p):
    """d_model 64: with and without the separator and the user embedding (negative user ids), H = 3, 5 and 8, histories full,
    end-padded, with holes, or with one fully masked."""
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, H=H, sep=sep, user_bins=user_bins, seed=H + 10 * sep).cuda().train()
    set_dropout(m, p)
    mask, ids, users = inputs(kind, 6, 5, H, 32, seed=H)
    assert (users < 0).any()
    batch = cuda_batch(batch_of(mask, ids, users, H, 32, seed=1))
    arms = tuple(ARMS) if p == 0.1 else tuple(a for a in ARMS if not ARMS[a][3])
    check_case(m, batch, p, f"small sep={sep} user_bins={user_bins} H={H} {kind} p={p}", arms, seed=H)


@pytest.mark.parametrize("attention", ["fp32", "tf32"])
def test_long_histories(attention):
    """8 histories of up to 200 items without the separator, with the user row: S = 601."""
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, sep=False, user_bins=7, seed=4).cuda().train()
    set_dropout(m, 0.1)
    mask, ids, users = inputs("holes", 8, 200, 3, 32, seed=8)
    batch = cuda_batch(batch_of(mask, ids, users, 3, 32, seed=2))
    check_case(m, batch, 0.1, "long", ("fused/fused" if attention == "fp32" else "fused/fused tf32",))


def test_relu_audit_at_the_measured_shape():
    """64 full 20-item histories without dropout, encoder="hf", decoder="fused": the shape at which the fused decoder's gradient
    was measured 1.8e-2 from HF's.  The pass is within the bounds of the statement that follows its relu decisions; the
    statement that follows its own float64 signs shows how far the flipped relus move a gradient, and it differs by more than
    the bound only where some relu flipped."""
    rs = np.random.RandomState(3)
    m = amazon().eval()
    batch = train_batch(rs, 64, 20, 3, 256)
    for arm in ("hf/fused", "fused/fused"):
        _, _, grads, flips = check_arm(m, batch, arm, 0.0, None, "measured shape")
        _, own = statement_grads(copy.deepcopy(m).double(), batch, None, None, 0.0)
        own_errs = grad_errors(grads, own)
        worst = max(own_errs, key=own_errs.get)
        print(f"measured shape [{arm}]: against the statement's own relu signs {own_errs[worst]:.2e} ({worst})")
        assert own_errs[worst] <= GRAD_BOUND or flips > 0, (arm, own_errs[worst])


def test_negative_controls():
    """Each wrong statement -- an attention site's keep bits from the next layer, a site without its 1/(1 - p), cross-attention
    bits at the packed row -- is at least ten times the bound away from the pass on some parameter."""
    from rq_vae_recommender_b200.modules import model as M
    m = random_model(M, H=3, sep=True, user_bins=7, seed=13).cuda().train()
    p = 0.1
    set_dropout(m, p)
    mask, ids, users = inputs("holes", 6, 5, 3, 32, seed=3)
    batch = cuda_batch(batch_of(mask, ids, users, 3, 32, seed=1))
    masks = Layout(m, batch).random_masks(m, p, 0)
    used, relus, grads, _ = check_arm(m, batch, "fused/fused", p, masks, "control")
    # HF-order encoder sites: 0 the embedding, then per layer l: 1 + 4l attention weights, 2 + 4l attention output, 3 + 4l
    # feed-forward inner, 4 + 4l feed-forward output
    next_layer = list(used)
    next_layer[1] = used[5]
    no_scale = list(used)
    no_scale[3] = used[3].double() * (1 - p)
    for what, kw in (("next layer's bits", dict(masks=next_layer)), ("no 1/(1 - p)", dict(masks=no_scale)),
                     ("packed-row cross bits", dict(masks=used, packed_row_bits=True))):
        _, wrong = statement_grads(copy.deepcopy(m).double(), batch, kw.pop("masks"), relus, p, **kw)
        errs = grad_errors(grads, wrong)
        worst = max(errs, key=errs.get)
        print(f"control {what}: {errs[worst]:.2e} ({worst}), {errs[worst] / GRAD_BOUND:.0f} x the bound")
        assert errs[worst] >= 10 * GRAD_BOUND, (what, errs[worst])
