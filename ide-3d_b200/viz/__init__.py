"""The visualizer's headless renderer (viz/renderer.py); the imgui/GLFW shell and its widgets are not part of this package."""
