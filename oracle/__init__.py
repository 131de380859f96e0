"""CPU oracle for the Precise streaming-inference hot path.  TEST INFRASTRUCTURE ONLY.

This package is a plain numpy restatement of the reference algorithm
(MycroftAI/mycroft-precise @ e1a635e) for the path

    int16 PCM -> MFCC (sonopy.mfcc_spec) -> GRU(h0=0, 29 steps) + Dense(1) + sigmoid
              -> ThresholdDecoder.decode -> TriggerDetector.update

Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference``
legs of ``bench.py`` may import it, and only as the checker / the CPU arm.  The product
(``mycroft_precise_b200``) never imports it and has no CPU fallback.

``cport.py`` / ``c/precise_oracle.c`` are a second, independent restatement of the same algorithm in plain C; the two
must agree (tests/test_oracle_c_port.py).

Parity pinning status
---------------------
* ``decoder.py``, ``trigger.py``, ``params.py``, ``listener.py`` (state machine): PINNED.  The
  reference's own ``precise/threshold_decoder.py``, ``precise/functions.py``,
  ``precise/params.py``, ``runner/precise_runner/runner.py`` and the real
  ``precise.network_runner.Listener`` class were imported unmodified from a reference checkout and their outputs committed as ``tests/golden/*.npz`` by
  ``tests/golden/make_golden.py``; ``tests/test_oracle_golden.py`` replays them.
* ``mfcc.py`` (sonopy 0.1.2, pinned in reference ``requirements.txt:35``) and ``gru.py``
  (Keras<=2.1.5 / TF 1.13 GRU+Dense, reference ``setup.py:75-78``): **PARITY UNPINNED**.
  Neither sonopy nor Keras/TF source is in the reference tree or installable for Python 3.12, and the reference's tests hold no golden vectors for this path
  (``test/scripts/test_engine.py:50`` asserts only an output regex).  These two files restate
  the published algorithms of those libraries; they are anchored on the reference's call
  sites (``precise/vectorization.py:36-39``, ``precise/model.py:77-82``), on analytic
  known-answer tests (all-zero / all-one frames, impulse, pure tone, hand-computed GRU steps)
  and on independent cross-checks (scipy.fftpack.dct, a direct O(N^2) DFT, a torch GRU cell
  rearranged to Keras semantics).
"""
