"""`python train.py algorithm=<ALG> env=<ENV> [key=value ...]` — same command line as the reference's train.py:21-23,
running the H100-native hot path (imitation-learning_b200/train.py). Multi-GPU: launch with torch.distributed.run."""
import il_b200  # noqa: F401
from il_b200.train import main

if __name__ == '__main__':
  main()
