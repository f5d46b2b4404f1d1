"""The draft rule of speculative decoding (speculative.cuh, spec_draft_kernel) and the pass counts it implies, restated in Python."""


def draft(emitted, prediction, prompt, max_draft, ngram):
    """Drafts of the next pass after `emitted`: for n = min(ngram, len(emitted)) down to 1, and for each source in order (the prediction,
    then, when `prompt` is not None, the prompt followed by the emitted tokens), the most recent occurrence of the last n emitted tokens
    that is followed by at least one token gives the up to max_draft tokens after it."""
    emitted = [int(t) for t in emitted]
    E = len(emitted)
    sources = [[int(t) for t in (prediction if prediction is not None else [])]]
    if prompt is not None:
        sources.append([int(t) for t in prompt] + emitted)
    for n in range(min(ngram, E), 0, -1):
        key = emitted[E - n:]
        for src in sources:
            for i in range(len(src) - n - 1, -1, -1):
                if src[i:i + n] == key:
                    return src[i + n:i + n + max_draft]
    return []


def simulate(output, prediction, prompt, max_draft, ngram):
    """(passes, drafted, accepted) of a request that emits `output` (its first token comes from the prefill): a pass emits the drafts that
    equal the request's own next tokens plus one token, cut where the output ends."""
    output = [int(t) for t in output]
    E, passes, drafted, accepted = 1, 0, 0, 0
    while E < len(output):
        d = draft(output[:E], prediction, prompt, max_draft, ngram)
        rem = len(output) - E
        j = 0
        while j < len(d) and j < rem and d[j] == output[E + j]:
            j += 1
        n = min(j + 1, rem)
        passes += 1
        drafted += len(d)
        accepted += min(j, n)
        E += n
    return passes, drafted, accepted
