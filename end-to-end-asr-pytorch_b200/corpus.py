"""LibriSpeech file listing (/root/reference/corpus/librispeech.py:28-61): glob the audio files of the splits, read
`<spk>-<chap>.trans.txt`, sort by token length, serve single items or buckets.  Out of the accelerated path; kept so
that `main.py --config <libri yaml>` is a drop-in."""
from pathlib import Path

from torch.utils.data import Dataset


def _transcripts(directory):
    table = {}
    for f in Path(directory).glob("*.trans.txt"):
        for line in open(f, "r"):
            utt, _, txt = line.rstrip("\n").partition(" ")
            table[utt] = txt
    return table


class LibriDataset(Dataset):
    def __init__(self, path, split, tokenizer, bucket_size, ascending=False):
        self.path, self.bucket_size = path, bucket_size
        files = []
        for s in split:
            found = sorted(list(Path(path, s).rglob("*.flac")) + list(Path(path, s).rglob("*.wav")))
            assert len(found) > 0, "No data found @ {}".format(Path(path, s))
            files += found
        cache = {}
        texts = []
        for f in files:
            d = str(f.parent)
            if d not in cache:
                cache[d] = _transcripts(d)
            texts.append(tokenizer.encode(cache[d][f.name.split(".")[0]]))
        pairs = sorted(zip(files, texts), reverse=not ascending, key=lambda x: len(x[1]))
        self.file_list, self.text = [p[0] for p in pairs], [p[1] for p in pairs]

    def __getitem__(self, index):
        if self.bucket_size > 1:
            index = min(len(self.file_list) - self.bucket_size, index)
            return list(zip(self.file_list[index:index + self.bucket_size], self.text[index:index + self.bucket_size]))
        return self.file_list[index], self.text[index]

    def __len__(self):
        return len(self.file_list)


# Official LibriSpeech LM text (corpus/librispeech.py:9-12 in the reference): read line by line, encoded on the fly, and
# the REMOVE_TOP_N_TXT longest lines dropped
OFFICIAL_TXT_SRC = ["librispeech-lm-norm.txt"]
REMOVE_TOP_N_TXT = 5000000


class LibriTextDataset(Dataset):
    """Sentences of LibriSpeech splits for the RNN LM (corpus/librispeech.py:64-122): transcripts found through the
    `*.flac` files of a split, and/or the lines of librispeech-lm-norm.txt.  All sentences are sorted by length,
    longest first (with the lm-norm file the length of the raw line, then the top REMOVE_TOP_N_TXT are dropped and
    every sentence is encoded when first served).  Files are listed in sorted path order."""

    def __init__(self, path, split, tokenizer, bucket_size):
        self.path, self.bucket_size = path, bucket_size
        self.encode_on_fly = False
        files, sents = [], []
        for s in split:
            if s in OFFICIAL_TXT_SRC:
                self.encode_on_fly = True
                with open(Path(path, s), "r") as f:
                    sents += f.readlines()
            files += sorted(Path(path, s).rglob("*.flac"))
        assert len(files) > 0 or len(sents) > 0, "No data found @ {}".format(path)
        cache = {}
        for f in files:
            d = str(f.parent)
            if d not in cache:
                cache[d] = _transcripts(d)
            sents.append(cache[d][f.name.split(".")[0]])
        if self.encode_on_fly:
            self.tokenizer = tokenizer
            self.text = sents
        else:
            self.text = [tokenizer.encode(t) for t in sents]
        self.text = sorted(self.text, reverse=True, key=len)
        if self.encode_on_fly:
            del self.text[:REMOVE_TOP_N_TXT]

    def _item(self, i):
        if self.encode_on_fly and type(self.text[i]) is str:
            self.text[i] = self.tokenizer.encode(self.text[i])
        return self.text[i]

    def __getitem__(self, index):
        if self.bucket_size > 1:
            index = min(len(self.text) - self.bucket_size, index)
            return [self._item(i) for i in range(index, index + self.bucket_size)]
        return self._item(index)

    def __len__(self):
        return len(self.text)
