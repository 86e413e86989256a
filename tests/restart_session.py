"""Session oracle with restarts: ``set_startpos`` on a live session.

``oracle.ltpl_session.OracleSession.set_startpos`` seeds the forced 'straight' memory of a FRESH session and keeps
everything else.  On a session that has already planned, the reference first drops its iterative memory
(OnlineTrajectoryHandler.reinit_iterative_memory, OTH:161-179, called at OTH:204 before the pose checks, so also for a
rejected pose); the next calc_paths is then a first tick again.  The calculation-time buffer (OTH:62), the trajectory id
base and the processed zone are not part of that memory and survive.  ``RestartSession`` restates exactly that on top
of ``OracleSession``; on a fresh session it behaves like its parent.
"""
from oracle.ltpl_session import OracleSession


class RestartSession(OracleSession):
    def set_startpos(self, pos, heading, vel=0.0):
        self.start_node = None
        self.m_nodes = self.m_node_idx = self.m_coeff = self.m_path = self.m_gg = self.m_red = self.m_bp = None
        self.last_path_timestamp = None
        self.last_cut_idx = 0
        self.pos_est = None
        self.backup = None
        return super().set_startpos(pos, heading, vel)
