#!/usr/bin/env python3
"""Generate noise_golden.npz from the REAL reference precise-add-noise (see make_golden.py for the other fixtures):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_noise_golden.py /path/to/mycroft-precise

Taken from the reference, unmodified: precise/scripts/add_noise.py's AddNoiseScript.run (tags file None), with its
NoiseData, TrainData.from_both / find_wavs, load_audio and save_audio, run after random.seed(SEED) on a small temporary
folder of seeded clips.  The image lacks the reference's command-line and audio packages, so ``prettyparse``, ``pyache`` and
``sonopy`` are stubs (nothing this script reaches uses them) and ``wavio`` is a stand-in on the stdlib ``wave`` module.

Recorded: the clips (in the order the script processed them, with their paths relative to the folder), the noise files in
the order NoiseData read them (one of them empty), each (file, copy)'s random() draw and noise ratio, the noise position
(in the noise files' cyclic concatenation) before each mix, the output paths relative to the output folder, and the
output samples as written.
"""
import argparse
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

SEED, INFLATION, LOW, HIGH = 7, 3, 0.1, 0.6

for name in ('prettyparse', 'pyache', 'sonopy'):
    stub = types.ModuleType(name)
    stub.Usage = lambda *a, **k: None
    stub.Pyache = object
    stub.mfcc_spec = stub.mel_spec = None
    sys.modules[name] = stub


class _Wav:
    def __init__(self, data, rate, sampwidth):
        self.data, self.rate, self.sampwidth = data, rate, sampwidth


def _read(file):
    with wave.open(file, 'rb') as w:
        data = np.frombuffer(w.readframes(w.getnframes()), '<i2').astype(np.int16)
        return _Wav(data.reshape(-1, w.getnchannels()), w.getframerate(), w.getsampwidth())


def _write(file, data, rate, sampwidth=2, scale=None):
    assert sampwidth == 2 and scale == 'none' and data.dtype == np.int16
    with wave.open(file, 'wb') as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(rate)
        w.writeframes(np.ascontiguousarray(data, '<i2').tobytes())


wavio = types.ModuleType('wavio')
wavio.Wav, wavio.read, wavio.write = _Wav, _read, _write
sys.modules['wavio'] = wavio

import precise.scripts.add_noise as an                                  # noqa: E402


def _save(path, pcm):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    _write(path, np.asarray(pcm, np.int16), 16000, 2, 'none')


def main():
    rs = np.random.RandomState(11)
    clip = lambda n, amp: np.clip(np.round(rs.randn(n) * amp), -32768, 32767).astype(np.int16)
    clips = {                                                      # every clip non-silent and well inside int16 range
        'wake-word/a.wav': clip(4000, 2500),
        'wake-word/sub/b.wav': clip(1601, 1800),
        'wake-word/c.wav': clip(12345, 3000),                      # longer than the whole noise corpus
        'not-wake-word/d.wav': clip(2, 1500),                       # (a 1-sample clip squeezes to a scalar there)
        'not-wake-word/e.wav': clip(777, 900),
        'test/wake-word/f.wav': clip(3333, 2000),
        'test/not-wake-word/g.wav': clip(2500, 1200),
    }
    noises = {'n1.wav': clip(5000, 2000), 'n2.wav': np.zeros(0, np.int16), 'n3.wav': clip(2100, 2600)}
    with tempfile.TemporaryDirectory() as tmp:
        folder, nfolder, ofolder = (os.path.join(tmp, d) for d in ('data', 'noise', 'out'))
        for rel, a in clips.items():
            _save(os.path.join(folder, rel), a)
        for rel, a in noises.items():
            _save(os.path.join(nfolder, rel), a)

        loaded, draws, positions, outputs = [], [], [], []
        load = an.load_audio
        an.load_audio = lambda f: loaded.append(f) or load(f)
        rnd = an.random
        an.random = lambda: draws.append(rnd()) or draws[-1]
        mix = an.NoiseData.noised_audio

        def noised_audio(self, audio, ratio):
            lens = [len(d) for d in self.noise_data]
            positions.append(sum(lens[:self.noise_data_id]) + self.noise_pos)
            return mix(self, audio, ratio)
        an.NoiseData.noised_audio = noised_audio
        save = an.save_audio
        an.save_audio = lambda f, a: outputs.append(f) or save(f, a)

        args = argparse.Namespace(folder=os.path.abspath(folder), tags_file=None, noise_folder=nfolder,
                                  output_folder=os.path.abspath(ofolder), inflation_factor=INFLATION,
                                  noise_ratio_low=LOW, noise_ratio_high=HIGH)
        random.seed(SEED)
        an.AddNoiseScript(args).run()

        noise_files = [f for f in loaded if f.startswith(nfolder)]
        clip_files = [f for f in loaded if f.startswith(folder + os.sep)]
        order = [os.path.relpath(f, folder) for f in clip_files]
        noise_order = [os.path.relpath(f, nfolder) for f in noise_files]
        out_names = [os.path.relpath(f, ofolder) for f in outputs]
        out_pcm = [np.squeeze(_read(f).data, 1) for f in outputs]
    ratios = np.asarray([LOW + (HIGH - LOW) * u for u in draws], np.float64)
    lens = np.asarray([len(o) for o in out_pcm], np.int64)
    np.savez_compressed(
        os.path.join(HERE, 'noise_golden.npz'),
        seed=np.int64(SEED), inflation=np.int64(INFLATION), low=np.float64(LOW), high=np.float64(HIGH),
        order=np.asarray(order), clip_pcm=np.concatenate([clips[r] for r in order]),
        clip_offsets=np.concatenate([[0], np.cumsum([len(clips[r]) for r in order])]).astype(np.int64),
        noise_order=np.asarray(noise_order), noise_pcm=np.concatenate([noises[r] for r in noise_order]),
        noise_offsets=np.concatenate([[0], np.cumsum([len(noises[r]) for r in noise_order])]).astype(np.int64),
        draws=np.asarray(draws, np.float64), ratios=ratios, positions=np.asarray(positions, np.int64),
        out_names=np.asarray(out_names), out_pcm=np.concatenate(out_pcm),
        out_offsets=np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
    print('wrote noise_golden.npz:', len(order), 'clips,', len(out_names), 'outputs; noise order', noise_order)


if __name__ == '__main__':
    main()
