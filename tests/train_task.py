"""The synthetic wake-word task the training tests share: a wake word is a rising chirp (600-1000 Hz, +1500 Hz/s, half a
second) somewhere in noise, a not-wake-word clip is the noise alone; clip lengths 12 000 .. 20 000 samples.  On the float64
restatement (oracle/train.py) an H = 20 network from GruModel.init(seed 0) trained for EPOCHS epochs of BATCH on 200 clips
scores at least MIN_ACCURACY on 200 held-out clips (tests/test_train_host.py), from about chance before training."""
import numpy as np

N_TRAIN, N_TEST = 200, 200
EPOCHS, BATCH = 8, 16
MIN_ACCURACY = 0.9


def clip(i, wake_word):
    rs = np.random.RandomState(5000 + i)
    n = rs.randint(12000, 20000)
    x = rs.randn(n) * 800
    if wake_word:
        f = 600 + 400 * rs.rand()
        a = rs.randint(0, n - 8000)
        t = np.arange(8000) / 16000
        x[a:a + 8000] += 6000 * np.sin(2 * np.pi * (f + 1500 * t) * t)
    return np.clip(x, -32768, 32767).astype(np.int16)


def dataset(first, n):
    """(clips, targets uint8): clips first .. first + n - 1, every other one a wake word."""
    clips = [clip(i, i % 2 == 0) for i in range(first, first + n)]
    return clips, np.asarray([i % 2 == 0 for i in range(first, first + n)], np.uint8)
