#!/usr/bin/env python3
"""Generate generated_golden.npz from the REAL reference precise-train-generated (see make_golden.py for the other fixtures):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_generated_golden.py /path/to/mycroft-precise

Taken from the reference, unmodified: precise/scripts/train_generated.py's TrainGeneratedScript.vectors_from_fn,
generate_wakeword_pieces, chunk_audio_pieces, layer_with, calc_volume, normalize_volume_to, merge and max_run_length, with
load_audio and chunk_audio, driven as generate_samples drives them (the shuffled background list cycled).  The instance is
made without __init__ (which builds a Keras model): the few attributes vectors_from_fn reads are set here as __init__ sets
them.  The image lacks Keras and the reference's command-line and audio packages, so ``keras``, ``fitipy``, ``prettyparse``,
``pyache`` and ``sonopy`` are stubs (nothing reached uses them) and ``wavio`` is a stand-in on the stdlib ``wave`` module.
The listener is a stub that records each merged chunk it is given, and the script's ``random`` records every draw.

To keep the fixture small the global ListenerParams runs at SAMPLE_RATE samples per second with a BUFFER_T second label
buffer, and chunks are CHUNK samples.  The clips hit all three cases of chunk_audio_pieces: a piece longer than a chunk
with a remainder, one an exact multiple of the chunk, and one shorter than a chunk.

Recorded: the background, wake-word and not-wake-word clips (in the order the run used them), the shuffled background order,
every random() draw in the order drawn, each merged chunk (float64) with its file and chunk index, and each chunk's decision
(1, 0, or -1 for a skipped window), for FILES background files (the list cycled, so vals_buffer carries across files).
"""
import os
import random
import sys
import tempfile
import types
import wave

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.dont_write_bytecode = True
REF = os.path.abspath(sys.argv[1])
sys.path.insert(0, REF)

SEED, SAMPLE_RATE, BUFFER_T, CHUNK, FILES, SAVE_PROB = 9, 4000, 0.75, 512, 9, 0.25


class _Usage:
    def __or__(self, other):
        return self


for name in ('prettyparse', 'pyache', 'sonopy', 'fitipy', 'keras', 'keras.callbacks'):
    stub = types.ModuleType(name)
    stub.Usage = lambda *a, **k: _Usage()
    stub.Pyache = stub.Fitipy = stub.LambdaCallback = object
    stub.mfcc_spec = stub.mel_spec = None
    sys.modules[name] = stub


class _Wav:
    def __init__(self, data, rate, sampwidth):
        self.data, self.rate, self.sampwidth = data, rate, sampwidth


def _read(file):
    with wave.open(file, 'rb') as w:
        data = np.frombuffer(w.readframes(w.getnframes()), '<i2').astype(np.int16)
        return _Wav(data.reshape(-1, w.getnchannels()), w.getframerate(), w.getsampwidth())


wavio = types.ModuleType('wavio')
wavio.Wav, wavio.read = _Wav, _read
sys.modules['wavio'] = wavio

from precise.params import pr                                          # noqa: E402
object.__setattr__(pr, 'sample_rate', SAMPLE_RATE)
object.__setattr__(pr, 'buffer_t', BUFFER_T)
import precise.scripts.train_generated as tg                           # noqa: E402


def _save(path, pcm):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with wave.open(path, 'wb') as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(SAMPLE_RATE)
        w.writeframes(np.ascontiguousarray(pcm, '<i2').tobytes())


class _Listener:
    def __init__(self):
        self.chunks = []

    def clear(self):
        pass

    def update_vectors(self, chunk):
        self.chunks.append(np.array(chunk, np.float64))
        return np.zeros((1, 1))


def main():
    rs = np.random.RandomState(17)
    sig = lambda n, amp: np.clip(np.round(rs.randn(n) * amp), -32768, 32767).astype(np.int16)
    backgrounds = [sig(n, a) for n, a in ((6000, 900), (4097, 1500), (12000, 400), (513, 1000))]
    wake = [sig(3500, 2500), sig(2 * CHUNK, 3000), sig(300, 2000), sig(6 * CHUNK, 2200)]
    other = [sig(700, 1200), sig(3 * CHUNK, 1800), sig(1900, 900)]
    with tempfile.TemporaryDirectory() as tmp:
        names = {}
        for kind, clips in (('bg', backgrounds), ('ww', wake), ('nww', other)):
            for i, a in enumerate(clips):
                p = os.path.join(tmp, kind, '%s%d.wav' % (kind, i))
                _save(p, a)
                names[p] = (kind, i)
        files = lambda kind: sorted(p for p, (k, _) in names.items() if k == kind)

        script = tg.TrainGeneratedScript.__new__(tg.TrainGeneratedScript)
        script.args = types.SimpleNamespace(chunk_size=CHUNK, save_prob=SAVE_PROB)
        script.audio_buffer = np.zeros(pr.buffer_samples, dtype=float)
        script.vals_buffer = np.zeros(pr.buffer_samples, dtype=float)
        script.listener = _Listener()
        script.pos_files_it = iter(tg.cycle(files('ww')))
        script.neg_files_it = iter(tg.cycle(files('nww')))

        draws, order, decisions = [], [], []
        rnd = tg.random
        tg.random = lambda: draws.append(rnd()) or draws[-1]
        saved = []
        tg.save_audio = lambda f, a: saved.append(f)
        random.seed(SEED)
        bg_files = files('bg')
        tg.shuffle(bg_files)
        order = [names[p][1] for p in bg_files]
        chunk_file, chunk_index = [], []
        for n in range(FILES):
            fn = bg_files[n % len(bg_files)]
            before = len(script.listener.chunks)
            kept = {}
            for mfccs, target in script.vectors_from_fn(fn):
                kept[len(script.listener.chunks) - 1] = target
            for j in range(before, len(script.listener.chunks)):
                decisions.append(kept.get(j, -1))
                chunk_file.append(n)
                chunk_index.append(j - before)
        chunks = script.listener.chunks
    cat = lambda clips: np.concatenate(clips)
    offs = lambda clips: np.concatenate([[0], np.cumsum([len(c) for c in clips])]).astype(np.int64)
    np.savez_compressed(
        os.path.join(HERE, 'generated_golden.npz'),
        seed=np.int64(SEED), sample_rate=np.int64(SAMPLE_RATE), buffer_samples=np.int64(pr.buffer_samples),
        chunk=np.int64(CHUNK), files=np.int64(FILES), save_prob=np.float64(SAVE_PROB),
        bg_pcm=cat(backgrounds), bg_offsets=offs(backgrounds), wake_pcm=cat(wake), wake_offsets=offs(wake),
        other_pcm=cat(other), other_offsets=offs(other), order=np.asarray(order, np.int64),
        draws=np.asarray(draws, np.float64), chunks=np.stack(chunks), decisions=np.asarray(decisions, np.int64),
        chunk_file=np.asarray(chunk_file, np.int64), chunk_index=np.asarray(chunk_index, np.int64),
        saved=np.int64(len(saved)))
    print('wrote generated_golden.npz: %d chunks, %d draws, decisions %s, %d saved' % (
        len(chunks), len(draws), np.bincount(np.asarray(decisions) + 1).tolist(), len(saved)))


if __name__ == '__main__':
    main()
