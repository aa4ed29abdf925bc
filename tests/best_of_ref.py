"""The temperature ladder with openai/whisper decode_with_fallback's choice of decoder per rung (test infrastructure, restated on top of
tests/language_ref.py's rung temperatures): beam search at temperature 0, best_of samples above it.  The library follows this rule when
DecodingOptions.bestOf is set; without it a beam call decodes one beam-search rung and any other call walks the plain ladder
(TranscribeTask.decodeWithFallback, TranscribeTask.swift:316-411)."""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

from oracle import decode_ref as D
from tests.language_ref import rung_temperatures


def rung_decoder(temperature: float, beamSize: int, bestOf: Optional[int]) -> Tuple[str, int]:
    """The decoder of one ladder rung and the rows it uses: ("beam", beamSize), ("best_of", bestOf) or ("single", 1).  bestOf None / 0
    keeps the library's plain rule (beam search on every rung of a beam call, else one row).  Otherwise openai/whisper's rule: beam
    search only at temperature 0 and only with beamSize > 1; independent samples only at temperature > 0 and only with bestOf > 1."""
    if beamSize > 1 and (not bestOf or temperature == 0.0):
        return "beam", beamSize
    if bestOf and bestOf > 1 and temperature > 0.0:
        return "best_of", bestOf
    return "single", 1


def ladder_plan(options: D.DecodingOptions, beamSize: int, bestOf: Optional[int]) -> List[Tuple[float, str, int]]:
    """(temperature, decoder, rows) of every rung a window may walk.  A beam call without bestOf has no ladder: one rung."""
    temps = rung_temperatures(options)
    if beamSize > 1 and not bestOf:
        temps = temps[:1]
    return [(t, *rung_decoder(t, beamSize, bestOf)) for t in temps]


def decode_with_fallback_best_of(decode_rung: Callable[[int, float, str, int], D.DecodingResult], options: D.DecodingOptions, beamSize: int,
                                 bestOf: Optional[int]):
    """The ladder with the per-rung decoder choice: decode_rung(rung, temperature, decoder, rows) returns that rung's chosen result
    (beam finalizer, best_of ranker or the single row).  The next rung runs while DecodingFallback asks for it.  Returns (result, rung)."""
    result, rung = None, 0
    for rung, (temp, kind, rows) in enumerate(ladder_plan(options, beamSize, bestOf)):
        result = decode_rung(rung, temp, kind, rows)
        if not (result.fallback is not None and result.fallback.needsFallback):
            break
    return result, rung
