"""Selection, bookkeeping and sharding logic of the outer loop — pure functions so that they can be
pinned by table tests (reference: tts/tts_reflectionflow.py:144-182,359-448) — plus the one
collective the sharded design adds: an all-gather of fixed-size score records per round
(SURVEY.md §8e)."""
from __future__ import annotations

import struct
from typing import Dict, List, Sequence, Tuple

import torch

MAX_SEED = 2 ** 31 - 1  # np.iinfo(np.int32).max (tts_reflectionflow.py:44)


# ------------------------------------------------------------------ sharding
def shard_candidates(num_candidates: int, rank: int, world: int) -> List[int]:
    """candidate i of a round -> rank i mod world (every rank derives the same table)."""
    return [i for i in range(num_candidates) if i % world == rank]


# ------------------------------------------------------------------ stub verifier
def stub_verifier_score(latents: torch.Tensor) -> torch.Tensor:
    """Deterministic scalar 'verifier' for offline runs: a fixed linear functional of the final
    latent evaluated in fp64 on the device (ties are measure-zero).  Returns [B] fp64."""
    x = latents.to(torch.float64).reshape(latents.shape[0], -1)
    n = x.shape[1]
    w = torch.cos(torch.arange(n, device=x.device, dtype=torch.float64) * 0.6180339887498949)
    return (x * w).sum(dim=1) / n


# ------------------------------------------------------------------ score exchange
RECORD_BYTES = 32  # cand_id:int32, label:int32, seed:int64, score:float64, pad


def pack_record(cand_id: int, seed: int, label: int, score: float) -> bytes:
    return struct.pack("<iiqd8x", int(cand_id), int(label), int(seed), float(score))


def unpack_record(b: bytes) -> Tuple[int, int, int, float]:
    cand_id, label, seed, score = struct.unpack("<iiqd8x", b)
    return cand_id, seed, label, score


def gather_records(local: Sequence[Tuple[int, int, int, float]], per_rank: int, rank: int,
                   world: int, device) -> List[Tuple[int, int, int, float]]:
    """One all-gather of `per_rank` fixed-size records from every rank (NCCL on GPUs, gloo on
    CPU).  Slots a rank does not fill carry cand_id = -1 and are dropped.  Every rank returns the
    same list, sorted by cand_id."""
    import torch.distributed as dist
    buf = bytearray()
    for i in range(per_rank):
        buf += pack_record(*local[i]) if i < len(local) else pack_record(-1, 0, 0, 0.0)
    t = torch.frombuffer(buf, dtype=torch.uint8).clone().to(device)
    if world > 1:
        out = torch.empty(world * t.numel(), dtype=torch.uint8, device=device)
        dist.all_gather_into_tensor(out, t)
    else:
        out = t
    raw = out.cpu().numpy().tobytes()
    recs = [unpack_record(raw[o:o + RECORD_BYTES]) for o in range(0, len(raw), RECORD_BYTES)]
    return sorted([r for r in recs if r[0] >= 0], key=lambda r: r[0])


def gather_scores(score: torch.Tensor, rank: int, world: int, device):
    """bench helper: one record per rank."""
    return gather_records([(rank, 0, 1, float(score.reshape(-1)[0].item()))], 1, rank, world, device)


# ------------------------------------------------------------------ selection rules (pinned by table tests)
def metric_value(output: dict, choice_of_metric: str):
    """tts_reflectionflow.py:152-155."""
    v = output[choice_of_metric]
    return v["score"] if isinstance(v, dict) else v


def nvila_key(output: dict):
    """tts_reflectionflow.py:165-169: "yes" first by descending score, then "no" by ascending."""
    return (0, -output["score"]) if output["label"] == "yes" else (1, output["score"])


METRIC_VERIFIERS = ("openai", "ours")  # ordered by outputs[choice_of_metric] (descending)


def sort_outputs(outputs: List[dict], verifier_name: str, choice_of_metric: str = None) -> List[dict]:
    if verifier_name in METRIC_VERIFIERS:
        return sorted(outputs, key=lambda x: metric_value(x, choice_of_metric), reverse=True)
    if verifier_name == "nvila":
        return sorted(outputs, key=nvila_key)
    raise NotImplementedError(f"Verifier {verifier_name} not supported")


def select_topk(outputs: List[dict], sorted_list: List[dict], items: list, topk: int):
    """tts_reflectionflow.py:175-182.  `outputs.index(x)` returns the FIRST equal dict, so equal
    score dicts collapse onto one index (SURVEY App. B.7) — kept on purpose."""
    topk_scores = sorted_list[:topk]
    topk_idx = [outputs.index(x) for x in topk_scores]
    selected = [items[i] for i in topk_idx]
    selected_outputs = [outputs[i] for i in topk_idx]
    if topk > len(selected):
        repeat = topk - len(selected)
        selected = selected + selected[:repeat]
        selected_outputs = selected_outputs + selected_outputs[:repeat]
        topk_idx = topk_idx + topk_idx[:repeat]
    return topk_idx, selected, selected_outputs


def compose_prompts(refined_prompt: List[str], reflections: List[str]) -> List[str]:
    """tts_reflectionflow.py:286-292."""
    if reflections:
        return [refined_prompt[i] + " [Reflexion]: " + reflections[i] for i in range(len(reflections))]
    return list(refined_prompt)


def update_chains(chains: Dict[str, dict], search_round: int, full_names: List[str],
                  outputs: List[dict], selected_parents: List[str], verifier_name: str,
                  choice_of_metric: str = None) -> Dict[str, dict]:
    """tts_reflectionflow.py:359-396, including the asymmetry that the nvila branch stops at the
    first chain containing the parent while the openai branch updates every such chain."""
    if verifier_name not in METRIC_VERIFIERS + ("nvila",):
        raise NotImplementedError(f"Verifier {verifier_name} not supported")
    metric = verifier_name in METRIC_VERIFIERS
    if search_round == 1:
        for i, name in enumerate(full_names):
            if name not in chains:
                chains[name] = {"images": [], "scores": []} if metric \
                    else {"images": [], "scores": [], "labels": []}
            chains[name]["images"].append(name)
            if metric:
                chains[name]["scores"].append(metric_value(outputs[i], choice_of_metric))
            else:
                chains[name]["labels"].append(outputs[i]["label"])
                chains[name]["scores"].append(outputs[i]["score"])
        return chains
    for i, name in enumerate(full_names):
        parent = selected_parents[i]
        for key in chains:
            if parent in chains[key]["images"]:
                chains[key]["images"].append(name)
                if metric:
                    chains[key]["scores"].append(metric_value(outputs[i], choice_of_metric))
                else:
                    chains[key]["labels"].append(outputs[i]["label"])
                    chains[key]["scores"].append(outputs[i]["score"])
                    break
    return chains


def best_per_chain(chains: Dict[str, dict], verifier_name: str) -> List[str]:
    """tts_reflectionflow.py:408-421."""
    best = []
    for chain in chains.values():
        if verifier_name in METRIC_VERIFIERS:
            scores = chain["scores"]
            idx = max(range(len(scores)), key=lambda j: (scores[j], -j))  # np.argmax: first max
        else:
            idx = min(range(len(chain["scores"])),
                      key=lambda j: (0 if chain["labels"][j] == "yes" else 1,
                                     -chain["scores"][j] if chain["labels"][j] == "yes"
                                     else chain["scores"][j]))
        best.append(chain["images"][idx])
    return best


def global_best(chains: Dict[str, dict], verifier_name: str) -> str:
    """tts_reflectionflow.py:428-446."""
    if verifier_name in METRIC_VERIFIERS:
        allv = [(s, n) for c in chains.values() for n, s in zip(c["images"], c["scores"])]
        return sorted(allv, key=lambda x: x[0], reverse=True)[0][1]
    allv = [(l, s, n) for c in chains.values()
            for n, l, s in zip(c["images"], c["labels"], c["scores"])]
    return sorted(allv, key=lambda x: (0 if x[0] == "yes" else 1, -x[1] if x[0] == "yes" else x[1]))[0][2]


# ---- parsers for the reflection generator's sectioned text (tts_reflectionflow.py:48-90; defined upstream but not
# called by the shipped loop — kept for callers that post-process reflections the same way)
def _reflection_items(content: str) -> List[str]:
    return [part.strip() for part in content.split("\n-") if part.strip()]


def extract_reflections(reflections: Sequence[str]) -> List[Dict[str, List[str]]]:
    """"<k>. <Title>:  <item>\\n- <item>..." sections separated by blank lines -> {title: [items]} per reflection
    (a section counts only if it has the colon + two spaces separator, :55-62)."""
    results = []
    for text in reflections:
        parsed: Dict[str, List[str]] = {}
        for section in text.split("\n\n"):
            if ":  " not in section:
                continue
            head, content = section.split(":  ", 1)
            parsed[head.split(". ", 1)[1].strip()] = _reflection_items(content)
        results.append(parsed)
    return results


def concat_extract_reflections(reflections: Sequence[str]) -> List[str]:
    """the items of every section joined by blanks, sections whose items mention "None" dropped, sections
    concatenated without a separator (:66-90)."""
    results = []
    for text in reflections:
        joined = ""
        for section in text.split("\n\n"):
            if ":" not in section:
                continue
            head, content = section.split(":", 1)
            head.split(".", 1)[1]  # the reference indexes the numbered title here too: un-numbered titles raise
            items = _reflection_items(content)
            if any("None" in item for item in items):
                continue
            joined += " ".join(items)
        results.append(joined)
    return results
