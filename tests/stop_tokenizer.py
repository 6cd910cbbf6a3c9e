"""A tokenizer built in-process from a seeded vocabulary (no tokenizer files are needed): a word-level model behind a
Metaspace pre-tokenizer / decoder, wrapped in PreTrainedTokenizerFast, so that pieces with a leading `▁` decode with a
leading space as sentencepiece pieces do.  Used by the stop-string tests and tools/bench_stop.py."""
import random

ALPHABET = 'ab#.xy'
# pieces every vocabulary starts with: the unknown token, the word transformers' StopStringCriteria.clean_tokenizer_vocab
# tokenizes as its static prefix, a piece whose string is empty, then pieces that contain, overhang or touch the stop
# strings the tests use
FIXED = ['<unk>', '▁abcdef', '', '#', '##', '###', '####', '▁#', '▁###', 'a#', '#b', 'x###y', '.###', '###.', 'a##', '#.',
         'a', 'b', 'ab', 'ba', 'abab', 'bab', 'aba', '▁ab', 'xab', 'aby', 'abx', 'x', 'y', '.', '▁']


def seeded_pieces(n, seed):
    """n distinct pieces: FIXED, then random strings of 1..6 characters of ALPHABET, a third of them with a leading `▁`."""
    rng = random.Random(seed)
    pieces, seen = list(FIXED), set(FIXED)
    while len(pieces) < n:
        p = ('▁' if rng.random() < 1 / 3 else '') + ''.join(rng.choice(ALPHABET) for _ in range(rng.randint(1, 6)))
        if p not in seen:
            seen.add(p)
            pieces.append(p)
    return pieces[:n]


def seeded_tokenizer(n, seed=0):
    """PreTrainedTokenizerFast over seeded_pieces(n, seed); piece i has id i."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    tk = Tokenizer(models.WordLevel({p: i for i, p in enumerate(seeded_pieces(n, seed))}, unk_token='<unk>'))
    tk.pre_tokenizer = pre_tokenizers.Metaspace()
    tk.decoder = decoders.Metaspace()
    return PreTrainedTokenizerFast(tokenizer_object=tk, unk_token='<unk>')
