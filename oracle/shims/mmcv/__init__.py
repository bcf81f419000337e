"""ORACLE / TEST INFRASTRUCTURE ONLY. Minimal stand-in for the un-vendored dependency named by the
package path (mmcv-full==1.5.3 / mmdet==2.25.0, environment.yml:27-28); restates only the
symbols imported at team_code_transfuser/model.py:20-30. parity unpinned (source absent)."""
