from buffalo_b200.evaluate.base import Evaluable
from buffalo_b200.evaluate.offline import evaluate_lists
