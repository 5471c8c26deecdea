"""Float64 CPU restatement of the bidirectional Lattice LSTM of model/lattice_lstm_crf.py, one sentence and one step at a
time (the shape of the public one-sentence implementation), so that autograd gives the reference gradients; and the
lattice word lists as a loop over substrings, the checker of the native builder."""
import torch

PARTS = ("char_cell", "word_cell", "alpha")


def names(scope="lattice_layer"):
    return {d: {p: (f"{scope}/{d}/{p}/kernel", f"{scope}/{d}/{p}/bias") for p in PARTS} for d in ("fw", "bw")}


def random_weights(Ec, Ew, H, seed, scale=1.0):
    """Glorot-uniform kernels and small random biases under the plugin's names (float32 CPU tensors)."""
    g = torch.Generator().manual_seed(seed)
    w = {}
    for d, parts in names().items():
        for p, (k, b) in parts.items():
            din, n = (Ew if p == "word_cell" else Ec) + H, (H if p == "alpha" else 3 * H)
            lim = (6.0 / (din + n)) ** 0.5 * scale
            w[k] = (torch.rand(din, n, generator=g) * 2 - 1) * lim
            w[b] = torch.randn(n, generator=g) * 0.1
    return w


def words_of(lens_row, n, Kw):
    """Valid words of one row: [(start, end, k)] for slots whose length is in [2, 10] and that end before n."""
    out = []
    for p in range(n):
        for k in range(Kw):
            ln = int(lens_row[p * Kw + k])
            if 2 <= ln <= 10 and p + ln - 1 < n:
                out.append((p, p + ln - 1, k))
    return out


def lattice_lstm(x, xw, lens, seq_len, w, H, alpha_shift=None):
    """x [B, L, Ec], xw [B, L, Kw, Ew] (slot embeddings), lens [B, L * Kw] int, seq_len [B], w: name -> tensor.
    -> out [B, L, 2H] in the dtype of x (use float64 tensors, with requires_grad where gradients are wanted).
    alpha_shift: optional [B, L, Kw, 2H] added to the alpha pre-activation of the word in slot (b, start, k), direction
    d at [..., d*H:(d+1)*H]; a zero leaf there collects each word's alpha gradient."""
    B, L, Ec = x.shape
    Kw, Ew = xw.shape[2], xw.shape[3]
    nm = names()
    zero = x.new_zeros(H)
    rows = []
    for b in range(B):
        n = max(0, min(int(seq_len[b]), L))
        words = words_of(lens[b], n, Kw)
        cols = []
        for di, d in enumerate(("fw", "bw")):
            Wc, bc = w[nm[d]["char_cell"][0]], w[nm[d]["char_cell"][1]]
            Ww, bw = w[nm[d]["word_cell"][0]], w[nm[d]["word_cell"][1]]
            Wa, ba = w[nm[d]["alpha"][0]], w[nm[d]["alpha"][1]]
            origin = (lambda wd: wd[0]) if di == 0 else (lambda wd: wd[1])
            target = (lambda wd: wd[1]) if di == 0 else (lambda wd: wd[0])
            h, c = zero, zero
            pending, outs = {}, [zero] * L
            for pos in (range(n) if di == 0 else range(n - 1, -1, -1)):
                z = x[b, pos] @ Wc[:Ec] + h @ Wc[Ec:] + bc
                i, o, g = torch.sigmoid(z[:H]), torch.sigmoid(z[H:2 * H]), torch.tanh(z[2 * H:])
                merged = [wd for wd in words if target(wd) == pos]
                if not merged:
                    c = (1 - i) * c + i * g
                else:
                    ei = torch.exp(i)
                    num, den = ei * g, ei
                    for wd in merged:
                        cw = pending.pop(wd)
                        za = x[b, pos] @ Wa[:Ec] + cw @ Wa[Ec:] + ba
                        if alpha_shift is not None:
                            za = za + alpha_shift[b, wd[0], wd[2], di * H:(di + 1) * H]
                        a = torch.sigmoid(za)
                        ea = torch.exp(a)
                        num, den = num + ea * cw, den + ea
                    c = num / den
                h = o * torch.tanh(c)
                outs[pos] = h
                for wd in words:
                    if origin(wd) == pos:
                        zw = xw[b, wd[0], wd[2]] @ Ww[:Ew] + h @ Ww[Ew:] + bw
                        pending[wd] = torch.sigmoid(zw[:H]) * c + torch.sigmoid(zw[H:2 * H]) * torch.tanh(zw[2 * H:])
            cols.append(torch.stack(outs))
        rows.append(torch.cat(cols, dim=-1))
    return torch.stack(rows)


def random_lattice(B, L, Kw, seq_len, seed, density=0.5, max_len=10):
    """Random slot lengths [B, L * Kw] int32: each slot filled with probability `density`, lengths 2..max_len (some
    reaching past seq_len, which the kernels must treat as empty)."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(2, max_len + 1, (B, L * Kw), generator=g, dtype=torch.int32)
    lens[torch.rand(B, L * Kw, generator=g) >= density] = 0
    return lens


def lattice_words(chars, vocab, max_seq_len, max_words, vocabfreq=None):
    """The lattice lists of one sentence (LatticeProc / ner_lexicon_build_lattice), written as the loop over substrings:
    for each start b < max_seq_len, the vocabulary words of 2..10 characters at [b, b + n) that end inside the first
    max_seq_len characters, in increasing length, then the max_words most frequent (stable sort).  vocab is a WordVocab.
    -> (ids [max_seq_len * max_words], lens [...], dropped); empty slots hold <PAD> and length 0."""
    vocabfreq = vocab.vocab_freq if vocabfreq is None else vocabfreq
    pad_id = vocab.vocab2idx[vocab.pad_token]
    n = min(len(chars), max_seq_len)
    ids, lens, dropped = [pad_id] * (max_seq_len * max_words), [0] * (max_seq_len * max_words), 0
    for b in range(n):
        found = []
        for e in range(b + 1, min(b + 10, n)):
            word = ''.join(chars[b:e + 1])
            if word in vocab.vocab2idx and vocab.vocab2idx[word] < vocab.n_word:
                found.append((vocab.vocab2idx[word], e - b + 1))
        if len(found) > max_words:
            dropped += len(found) - max_words
            found = sorted(found, key=lambda t: vocabfreq.get(t[0], 1), reverse=True)[:max_words]
        for k, (i, ln) in enumerate(found):
            ids[b * max_words + k], lens[b * max_words + k] = i, ln
    return ids, lens, dropped
