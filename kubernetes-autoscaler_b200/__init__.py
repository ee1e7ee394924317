"""caengine — H100-native scale-up simulation engine for the Cluster Autoscaler hot path.

Import as ``kubernetes_autoscaler_b200`` (alias package at the repo root)."""
