"""H100-native fused tri-plane volume renderer (drop-in for the render path of
google-research/nerf-from-image).  See README.md."""
