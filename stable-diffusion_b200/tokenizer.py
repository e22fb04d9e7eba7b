"""CLIP byte-level BPE tokenizer on the host (SURVEY 8 a18: `FrozenCLIPEmbedder.forward` = tokenizer(text,
truncation=True, max_length=77, padding="max_length") -> input_ids, ldm/modules/encoders/modules.py:153-156).

The reference delegates to `transformers.CLIPTokenizer` (third-party, version pinned by environment.yaml:26) and its
vocabulary files (`vocab.json`, `merges.txt` of openai/clip-vit-large-patch14). This is a dependency-free restatement
of the published algorithm so prompts can be encoded from those two files alone:
  NFC -> collapse whitespace -> lowercase -> split with the CLIP pattern -> bytes mapped to printable code points ->
  byte-pair merges by rank with the end-of-word marker `</w>` -> ids; [BOS] + 75 tokens max + [EOS], padded with EOS.
It is pinned against the installed `transformers.CLIPTokenizer` on a synthetic vocabulary (tests/test_tokenizer_cpu.py);
no real vocabulary ships offline, so the files have to be supplied by the user (a directory with both files).
"""
from __future__ import annotations

import json
import os
import unicodedata

try:
    import regex as _regex
    _PAT = _regex.compile(r"""'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""")
except ImportError:   # the scanner below implements the same pattern with unicodedata (stdlib `re` has no \p{L} / \p{N}:
    _regex = None     # its \d / [^\W\d_] approximations glue characters such as '²', '½', 'Ⅳ' to neighbouring words)
    _PAT = None

_CONTRACTIONS = ("'s", "'t", "'re", "'ve", "'m", "'ll", "'d")
# \s of the `regex` / Rust regex engines = the Unicode White_Space property
_WHITE = frozenset("\t\n\x0b\x0c\r \x85\xa0\u1680\u2000\u2001\u2002\u2003\u2004\u2005\u2006\u2007\u2008\u2009\u200a"
                   "\u2028\u2029\u202f\u205f\u3000")


def _is_letter(ch):
    return unicodedata.category(ch)[0] == "L"


def _is_number(ch):
    return unicodedata.category(ch)[0] == "N"


def split_clip(text):
    """The CLIP pre-tokenisation pattern  's|'t|'re|'ve|'m|'ll|'d|[\\p{L}]+|[\\p{N}]|[^\\s\\p{L}\\p{N}]+  as a scanner over
    Unicode general categories (leftmost match, alternatives tried in order, exactly as the regex does)."""
    out, i, n = [], 0, len(text)
    while i < n:
        ch = text[i]
        if ch == "'":
            hit = next((c for c in _CONTRACTIONS if text.startswith(c, i)), None)
            if hit:
                out.append(hit)
                i += len(hit)
                continue
        if _is_letter(ch):
            j = i + 1
            while j < n and _is_letter(text[j]):
                j += 1
        elif _is_number(ch):
            j = i + 1
        elif ch in _WHITE:
            i += 1
            continue
        else:
            j = i + 1
            while j < n and not (text[j] in _WHITE or _is_letter(text[j]) or _is_number(text[j])):
                j += 1
        out.append(text[i:j])
        i = j
    return out


def _collapse_white(text):
    """Replace(Regex(r"\\s+"), " ") of the reference tokenizer's normaliser."""
    out, prev = [], False
    for ch in text:
        if ch in _WHITE:
            if not prev:
                out.append(" ")
            prev = True
        else:
            out.append(ch)
            prev = False
    return "".join(out)


BOS, EOS = "<|startoftext|>", "<|endoftext|>"


def bytes_to_unicode():
    """The GPT-2 / CLIP byte -> printable code point table (bytes that are printable map to themselves)."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("\xa1"), ord("\xac") + 1)) + list(range(ord("\xae"), ord("\xff") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return {b: chr(c) for b, c in zip(bs, cs)}


class CLIPBPETokenizer:
    def __init__(self, vocab, merges, max_length=77):
        """vocab: {token: id} or a path to vocab.json; merges: ["a b", ...] in rank order or a path to merges.txt."""
        if isinstance(vocab, (str, os.PathLike)):
            with open(vocab, encoding="utf-8") as f:
                vocab = json.load(f)
        if isinstance(merges, (str, os.PathLike)):
            with open(merges, encoding="utf-8") as f:
                lines = f.read().split("\n")
            merges = [ln for ln in lines if ln and not ln.startswith("#version")]
        self.vocab = dict(vocab)
        self.ranks = {}
        for i, m in enumerate(merges):
            a, b = m.split(" ") if isinstance(m, str) else m
            self.ranks.setdefault((a, b), i)
        self.byte_encoder = bytes_to_unicode()
        self.max_length = max_length
        self.bos_id, self.eos_id = self.vocab[BOS], self.vocab[EOS]
        self.unk_id = self.eos_id            # unk_token = "<|endoftext|>" in the CLIP tokenizer config
        self._cache = {}

    @classmethod
    def from_dir(cls, path, max_length=77):
        return cls(os.path.join(path, "vocab.json"), os.path.join(path, "merges.txt"), max_length)

    def __len__(self):
        return len(self.vocab)

    # -- byte-pair merges of one pre-token (already byte-mapped), end-of-word marker on its last symbol
    def _bpe(self, token):
        hit = self._cache.get(token)
        if hit is not None:
            return hit
        word = list(token[:-1]) + [token[-1] + "</w>"]
        while len(word) > 1:
            best, best_rank = None, None
            for i in range(len(word) - 1):
                r = self.ranks.get((word[i], word[i + 1]))
                if r is not None and (best_rank is None or r < best_rank):
                    best, best_rank = (word[i], word[i + 1]), r
            if best is None:
                break
            merged, i = [], 0
            while i < len(word):
                if i < len(word) - 1 and word[i] == best[0] and word[i + 1] == best[1]:
                    merged.append(best[0] + best[1])
                    i += 2
                else:
                    merged.append(word[i])
                    i += 1
            word = merged
        self._cache[token] = word
        return word

    def _encode_plain(self, text):
        text = _collapse_white(unicodedata.normalize("NFC", text)).lower()
        ids = []
        for tok in (_PAT.findall(text) if _PAT is not None else split_clip(text)):
            mapped = "".join(self.byte_encoder[b] for b in tok.encode("utf-8"))
            ids.extend(self.vocab.get(piece, self.unk_id) for piece in self._bpe(mapped))
        return ids

    def tokenize_ids(self, text):
        """Token ids of `text` without BOS / EOS / padding; the two special-token literals map to their ids."""
        ids, rest = [], text
        while rest:
            cut = min((rest.find(s) for s in (BOS, EOS) if s in rest), default=-1)
            if cut < 0:
                ids.extend(self._encode_plain(rest))
                break
            ids.extend(self._encode_plain(rest[:cut]))
            special = BOS if rest.startswith(BOS, cut) else EOS
            ids.append(self.vocab[special])
            rest = rest[cut + len(special):]
        return ids

    def __call__(self, texts, max_length=None):
        """list[str] (or one str) -> list of max_length-long id lists: BOS + tokens (truncated) + EOS, EOS padding."""
        if isinstance(texts, str):
            texts = [texts]
        n = max_length or self.max_length
        out = []
        for t in texts:
            ids = [self.bos_id] + self.tokenize_ids(t)[: n - 2] + [self.eos_id]
            out.append(ids + [self.eos_id] * (n - len(ids)))
        return out


# ------------------------------------------------------------------------------------------------ BERT WordPiece
# `BERTTokenizer` of the LAION-400M model (ldm/modules/encoders/modules.py:53-67) is transformers' BertTokenizerFast
# ("bert-base-uncased") with truncation to 77 and max_length padding. The restatement below follows the published
# uncased BERT pipeline from a vocab.txt alone:
#   raw text split on the literal special tokens -> drop NUL / U+FFFD / control characters, whitespace to " " -> spaces
#   around CJK ideographs -> NFD and drop non-spacing marks -> lowercase -> split on whitespace, every punctuation
#   character a token of its own -> greedy longest-match WordPiece ("##" continuation, [UNK] for a word that does not
#   decompose or is longer than 100 characters) -> [CLS] + 75 tokens max + [SEP], padded with [PAD].
# It is pinned against the installed transformers.BertTokenizerFast on a synthetic vocabulary (tests/test_laion_cpu.py).
BERT_SPECIAL = ("[CLS]", "[SEP]", "[PAD]", "[UNK]", "[MASK]")


def _bert_is_white(ch):
    return ch in "\t\n\r" or ch in _WHITE


def _bert_is_control(ch):
    return ch not in "\t\n\r" and unicodedata.category(ch)[0] == "C"


def _bert_is_punct(ch):
    o = ord(ch)
    return 33 <= o <= 47 or 58 <= o <= 64 or 91 <= o <= 96 or 123 <= o <= 126 or unicodedata.category(ch)[0] == "P"


def _is_cjk(ch):
    o = ord(ch)
    return (0x4E00 <= o <= 0x9FFF or 0x3400 <= o <= 0x4DBF or 0x20000 <= o <= 0x2A6DF or 0x2A700 <= o <= 0x2B73F or
            0x2B740 <= o <= 0x2B81F or 0x2B920 <= o <= 0x2CEAF or 0xF900 <= o <= 0xFAFF or 0x2F800 <= o <= 0x2FA1F)


def bert_normalize(text):
    """The uncased BERT normaliser: clean-up, CJK spacing, accent stripping, per-character lowercasing."""
    out = []
    for ch in text:
        if ch == "\x00" or ch == "�" or _bert_is_control(ch):
            continue
        if _bert_is_white(ch):
            out.append(" ")
        elif _is_cjk(ch):
            out.append(" " + ch + " ")
        else:
            out.append(ch)
    text = unicodedata.normalize("NFD", "".join(out))
    return "".join(ch.lower() for ch in text if unicodedata.category(ch) != "Mn")


def bert_split(text):
    """Whitespace splits (and is dropped); each punctuation character is a word of its own."""
    words, cur = [], []
    for ch in text:
        if _bert_is_white(ch) or _bert_is_punct(ch):
            if cur:
                words.append("".join(cur))
                cur = []
            if not _bert_is_white(ch):
                words.append(ch)
        else:
            cur.append(ch)
    if cur:
        words.append("".join(cur))
    return words


class BertWordPieceTokenizer:
    def __init__(self, vocab, max_length=77, max_word_chars=100):
        """vocab: {token: id} or a path to vocab.txt (one token per line, id = line number)."""
        if isinstance(vocab, (str, os.PathLike)):
            with open(vocab, encoding="utf-8") as f:
                vocab = {ln.rstrip("\n"): i for i, ln in enumerate(f) if ln.rstrip("\n")}
        self.vocab = dict(vocab)
        missing = [t for t in ("[CLS]", "[SEP]", "[PAD]", "[UNK]") if t not in self.vocab]
        if missing:
            raise ValueError(f"BERT vocabulary lacks {missing}")
        self.cls_id, self.sep_id = self.vocab["[CLS]"], self.vocab["[SEP]"]
        self.pad_id, self.unk_id = self.vocab["[PAD]"], self.vocab["[UNK]"]
        self.max_length, self.max_word_chars = max_length, max_word_chars
        self._specials = [t for t in BERT_SPECIAL if t in self.vocab]

    @classmethod
    def from_dir(cls, path, max_length=77):
        return cls(os.path.join(path, "vocab.txt"), max_length)

    def __len__(self):
        return len(self.vocab)

    def _wordpiece(self, word):
        if len(word) > self.max_word_chars:
            return [self.unk_id]
        ids, start = [], 0
        while start < len(word):
            end = len(word)
            while end > start:
                piece = word[start:end] if start == 0 else "##" + word[start:end]
                if piece in self.vocab:
                    ids.append(self.vocab[piece])
                    break
                end -= 1
            if end == start:
                return [self.unk_id]
            start = end
        return ids

    def _encode_plain(self, text):
        ids = []
        for w in bert_split(bert_normalize(text)):
            ids.extend(self._wordpiece(w))
        return ids

    def tokenize_ids(self, text):
        """Token ids of `text` without [CLS] / [SEP] / padding; literal special tokens map to their ids."""
        ids, rest = [], text
        while rest:
            hits = [(rest.find(s), s) for s in self._specials if s in rest]
            if not hits:
                ids.extend(self._encode_plain(rest))
                break
            cut, special = min(hits, key=lambda h: (h[0], -len(h[1])))
            ids.extend(self._encode_plain(rest[:cut]))
            ids.append(self.vocab[special])
            rest = rest[cut + len(special):]
        return ids

    def __call__(self, texts, max_length=None):
        """list[str] (or one str) -> list of max_length-long id lists: [CLS] + tokens (truncated) + [SEP], [PAD] after."""
        if isinstance(texts, str):
            texts = [texts]
        n = max_length or self.max_length
        out = []
        for t in texts:
            ids = [self.cls_id] + self.tokenize_ids(t)[: n - 2] + [self.sep_id]
            out.append(ids + [self.pad_id] * (n - len(ids)))
        return out
