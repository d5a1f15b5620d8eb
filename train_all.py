"""`python train_all.py algorithm=<ALG> [key=value ...]` trains one configuration on every env and returns the minimum over envs of its score;
`python train_all.py -m algorithm=<ALG> [fixed key=value ...] [hpo.<key>=value ...]` searches conf/hyperparameter_search_space/<ALG>.yaml
(imitation-learning_b200/hpo.py). Same command line as the reference's train_all.py."""
import il_b200  # noqa: F401
from il_b200.hpo import main

if __name__ == '__main__':
  main()
