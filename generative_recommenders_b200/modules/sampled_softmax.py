"""Sampled-softmax training loss on the H100 ops (SURVEY.md section 8 row f3).

Mirrors generative_recommenders/research/modeling/sequential/losses/sampled_softmax.py:29-193 (`SampledSoftmaxLoss`) and the
sampler it is configured with, autoregressive_losses.py:29-121 (`NegativesSampler`, `LocalNegativesSampler`): same constructor
arguments, same random draw (`torch.randint(0, num_items, ids.shape + (R,))` on the device of the ids, so a seeded run samples
the ids the reference samples), same loss.  The similarity is the dot product the reference configures for HSTU
(rails/similarities/dot_product_similarity_fn.py): with a `LocalNegativesSampler` the loss runs as ONE fused kernel that reads
the R negative rows of every query straight from the item table instead of materialising [N, R, D].
"""
from typing import Dict, List, Tuple

import torch

from ..ops.sampled_softmax import sampled_softmax_loss


class LocalNegativesSampler(torch.nn.Module):
    def __init__(self, num_items: int, item_emb: torch.nn.Embedding, all_item_ids: List[int], l2_norm: bool,
                 l2_norm_eps: float) -> None:
        super().__init__()
        self._l2_norm, self._l2_norm_eps = l2_norm, l2_norm_eps
        self._num_items: int = len(all_item_ids)
        self._item_emb: torch.nn.Embedding = item_emb
        self.register_buffer("_all_item_ids", torch.tensor(all_item_ids))

    def debug_str(self) -> str:
        return f"local{f'-l2-eps{self._l2_norm_eps}' if self._l2_norm else ''}"

    def process_batch(self, ids, presences, embeddings) -> None:
        pass

    def normalize_embeddings(self, x: torch.Tensor) -> torch.Tensor:
        if self._l2_norm:
            x = x / torch.clamp(torch.linalg.norm(x, ord=2, dim=-1, keepdim=True), min=self._l2_norm_eps)
        return x

    def sample_ids(self, positive_ids: torch.Tensor, num_to_sample: int) -> torch.Tensor:
        """The id half of the reference's forward (autoregressive_losses.py:106-121): same generator call, same shapes."""
        output_shape = positive_ids.size() + (num_to_sample,)
        sampled_offsets = torch.randint(low=0, high=self._num_items, size=output_shape, dtype=positive_ids.dtype,
                                        device=positive_ids.device)
        return self._all_item_ids[sampled_offsets.view(-1)].reshape(output_shape)

    def forward(self, positive_ids: torch.Tensor, num_to_sample: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """(sampled_ids, sampled_negative_embeddings) like the reference; SampledSoftmaxLoss does not call this (it never
        gathers the embeddings), it is kept for callers that want the tensors."""
        sampled_ids = self.sample_ids(positive_ids, num_to_sample)
        return sampled_ids, self.normalize_embeddings(self._item_emb(sampled_ids))


class SampledSoftmaxLoss(torch.nn.Module):
    def __init__(self, num_to_sample: int, softmax_temperature: float, model=None, activation_checkpoint: bool = False) -> None:
        super().__init__()
        self._num_to_sample: int = num_to_sample
        self._softmax_temperature: float = softmax_temperature
        self._model = model  # the reference reads model.similarity_fn; here the similarity is the (fused) dot product
        self._activation_checkpoint: bool = activation_checkpoint  # nothing to checkpoint: [N, R, D] is never materialised

    def jagged_forward(self, output_embeddings: torch.Tensor, supervision_ids: torch.Tensor, supervision_embeddings: torch.Tensor,
                       supervision_weights: torch.Tensor, negatives_sampler: LocalNegativesSampler,
                       **kwargs) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        assert output_embeddings.size() == supervision_embeddings.size()
        assert supervision_ids.size() == supervision_embeddings.size()[:-1]
        assert supervision_ids.size() == supervision_weights.size()
        if not isinstance(negatives_sampler, LocalNegativesSampler):
            raise NotImplementedError("the fused CUDA loss needs a LocalNegativesSampler (ids into one embedding table)")
        sampled_ids = negatives_sampler.sample_ids(positive_ids=supervision_ids, num_to_sample=self._num_to_sample)
        loss = sampled_softmax_loss(output_embeddings, supervision_ids, supervision_embeddings, supervision_weights, sampled_ids,
                                    negatives_sampler._item_emb.weight, self._softmax_temperature, negatives_sampler._l2_norm,
                                    negatives_sampler._l2_norm_eps)
        return loss, {}

    def forward(self, lengths: torch.Tensor, output_embeddings: torch.Tensor, supervision_ids: torch.Tensor,
                supervision_embeddings: torch.Tensor, supervision_weights: torch.Tensor, negatives_sampler: LocalNegativesSampler,
                **kwargs) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        """Dense [B, N, ...] inputs with `lengths` valid positions per row (sampled_softmax.py:91-193): the first lengths[b]
        positions of every row are kept (dense_to_jagged) and the jagged loss is evaluated on them."""
        torch._assert(output_embeddings.size() == supervision_embeddings.size(), "Invalid supervision embeddings size.")
        torch._assert(supervision_ids.size() == supervision_embeddings.size()[:-1], "Invalid supervision ids size.")
        B, N = supervision_ids.shape
        keep = torch.arange(N, device=lengths.device).unsqueeze(0) < lengths.unsqueeze(1)  # [B, N]
        return self.jagged_forward(output_embeddings=output_embeddings[keep], supervision_ids=supervision_ids[keep],
                                   supervision_embeddings=supervision_embeddings[keep],
                                   supervision_weights=supervision_weights[keep], negatives_sampler=negatives_sampler, **kwargs)
