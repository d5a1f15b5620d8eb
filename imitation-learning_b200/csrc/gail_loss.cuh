// The GAIL discriminator's loss and reward (training.py:94-114,130-132; models.py:177-180), written once for the fused depth-1 kernels
// (gail.cu) and the general program (gail_general.cu).
#pragma once
#include "common.cuh"

// One pass of a discriminator update: the rows it reads and the loss terms its logits take. PASS_ANY (-1) marks work every replica shares.
enum PassKind { PASS_ANY = -1, PASS_POLICY = 0, PASS_EXPERT = 1, PASS_MIX = 2, PASS_PENALTY = 3 };

// PUGAIL's clamp (training.py:102) from the batch sums of w softplus(f) over the policy and expert rows: torch.clamp(min=) passes gradient
// where x >= min, so 1 keeps the gated terms and 0 drops them (the policy loss is then -margin).
__device__ __forceinline__ float gail_pu_gate(float sum_policy, float sum_expert, float prior, float margin, float invB) {
  return (prior * (sum_expert * invB) - sum_policy * invB) >= -margin ? 1.f : 0.f;
}

// dL/dlogit of one row of weight w and logit f; adds the row's loss term to `loss`. mix: a Mixup row with mixing epsilon e; otherwise a BCE or
// PUGAIL row of the expert (expert) or policy batch.
__device__ __forceinline__ float gail_loss_row(float f, float w, bool mix, float e, int loss_function, bool expert, float prior, float pu_gate,
                                               float entropy_bonus, float invB, float& loss) {
  const float sg = sigmoidf(f);
  float df;
  if (mix) {  // training.py:112
    df = w * (sg - e) * invB;
    loss += e * w * softplusf(-f) + (1.f - e) * w * softplusf(f);
  } else if (loss_function == IL_LOSS_BCE) {  // training.py:98-99
    df = expert ? w * (sg - 1.f) * invB : w * sg * invB;
    loss += expert ? w * softplusf(-f) : w * softplusf(f);
  } else {  // PUGAIL, training.py:101-102
    const float pr = prior;
    df = expert ? pr * w * (sg - 1.f) * invB + pu_gate * pr * w * sg * invB : -pu_gate * w * sg * invB;
    loss += expert ? pr * w * softplusf(-f) + pu_gate * pr * w * softplusf(f) : -pu_gate * w * softplusf(f);
  }
  if (entropy_bonus > 0.f) df += entropy_bonus * w * f * sg * (1.f - sg) * invB;  // training.py:130-132
  return df;
}

// The reward of a logit (models.py:177-180).
__device__ __forceinline__ float gail_reward_of_logit(float f, int reward_function) {
  const float D = sigmoidf(f);
  float h = reward_function == IL_REWARD_GAIL ? -log1pf(-D + 1e-6f) : logf(D + 1e-6f) - log1pf(-D + 1e-6f);
  if (reward_function == IL_REWARD_FAIRL) h = expf(h) * -h;
  return h;
}
